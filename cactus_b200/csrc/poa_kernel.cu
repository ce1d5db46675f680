// poa_kernel.cu -- the fused, batched partial-order-alignment kernel for sm_90a (H100).
//
// One CTA owns one job (= one abpoa_msa call of the reference: K sequences -> one MSA) from start to finish:
// it keeps the job's partial-order graph in its slot of device memory, aligns the sequences to it one after the
// other and never returns to the host in between. CTAs are persistent: each pulls the next job index from a
// global counter, so a launch of (SMs x resident CTAs) blocks streams through thousands of jobs while the
// strictly sequential phases of some jobs (traceback, graph fusion, topological sort) overlap the DP sweeps of
// the other CTAs resident on the same SM.
//
// DP sweep (the hot loop; replaces simd_abpoa_cg_dp + first row + row max + adaptive band,
// abPOA src/abpoa_align_simd.c:617-688, 935-1130):
//   * graph rows in topological order, strictly one after the other (the adaptive band of a row needs the argmax
//     columns of all predecessor rows); the columns of a row in parallel;
//   * column ownership is FIXED: thread t owns columns [16t, 16t+16) of every row. The H / E1 / E2 values of the
//     row just computed therefore stay in the owning thread's registers and feed the next row without touching
//     memory when the predecessor is the previous row (the common case in a near-linear graph); only H[16t-1]
//     comes from the neighbour thread (warp shuffle; one shared-memory word per warp boundary). Predecessors
//     two rows back (every substitution bubble and deletion makes such rows) are read from a ring of the last two rows in
//     the CTA's dynamic shared memory, where the class's scratch holds two rows; older ones from the planes in global memory
//     (L2), one 16-byte chunk per thread and instruction, a warp's chunk 512 contiguous bytes;
//   * the max-plus recurrence of the two insertion states F1/F2 along the row is turned into a plain prefix
//     maximum by the substitution A[k] = H'[k] - oe + (k+1)*e  =>  F[j] = max_{k<j} A[k] - j*e across threads: a warp
//     shuffle scan over the 32 thread aggregates, a redux over the warp aggregates staged in shared memory. Within a
//     thread's 16 cells the recurrence itself runs, one add-max per cell and plane (row_pass1, row_pass2);
//   * per cell the sweep writes 8 bytes for the traceback and for later rows -- H (int32) and the two E values as 16-bit
//     distances below H; F1 / F2 are not stored, the traceback recomputes the few row prefixes it needs
//     (poa_types.h: DpState) -- in a chunk-major layout where every 128-bit warp store writes 512 contiguous bytes:
//     8 B/cell of HBM write traffic (the reference streams five int32 planes, 20 B/cell) is the kernel's only DRAM stream;
//   * two block barriers per row.
// Integer DP: no tensor cores. int32 everywhere with the reference's own "minus infinity" so that finite cells
// are bit-identical to abPOA's AVX2 path.
#include <cuda_runtime.h>
#include <stdint.h>
#include "poa_graph.cuh"
#include "poa_cta.cuh"
#include "poa_kernel.cuh"

namespace barb200 {

#define FULL 0xffffffffu

struct KShared {
    Graph g; RowTables rt; DpState d;
    int job, msa_len_s, abort_s;
    // [graph base][query code 0..4, 5 = "no base": column 0 / beyond the query -> 0]. 256-byte aligned: the sweep forms an
    // entry's shared-memory address by replacing the low byte of the table's with the byte offset 32 * base + 4 * code
    __align__(256) int smat[5 * 8];
    int wF[2][2][32];      // [row parity][plane F1/F2][warp] block scan staging
    int wM[2][4][32];      // [row parity][max, leftmost, rightmost, H of the warp's last column][warp]
    RowRec rec[2];         // [row parity] the sweep's row record, fetched one row ahead
    RowInfo ring_info[2];  // [row parity] band of the row held in that slot of the shared-memory ring (dp_sweep)
};

__device__ __forceinline__ int4 ld4cg(const int *p) { return __ldcg(reinterpret_cast<const int4 *>(p)); }
// one 128-bit store per plane chunk: a warp's store writes 512 contiguous bytes, 4 whole lines, in one instruction. An int4
// assignment is split into four 32-bit stores by NVVM in this kernel, and each of those spans the same 4 lines. The PTX store
// keeps the default cache policy: far-predecessor rows are read back from L2 a few rows after they are written.
// tests/test_sweep_sass.py pins every store of this helper to STG.E.128
__device__ __forceinline__ void st4(int *p, int a, int b, int c, int d) {
    asm volatile("st.global.v4.s32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
// the same 16-byte chunks in the shared-memory ring of the sweep: one STS.128 / LDS.128 per chunk, a warp's access 512
// contiguous bytes (conflict-free); tests/test_sweep_ring_sass.py pins them. a: shared-window byte address
__device__ __forceinline__ void sts4(unsigned a, int x, int y, int z, int w) {
    asm volatile("st.shared.v4.s32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ int4 lds4(unsigned a) {
    int4 v;
    asm volatile("ld.shared.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ int lds1(unsigned a) {
    int v;
    asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
// a load from a table in shared memory that does not change while the sweep runs: not volatile, so that the compiler can
// schedule the loads of a row's cells freely
__device__ __forceinline__ int lds_const(unsigned a) {
    int v;
    asm("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ int max3(int a, int b, int c) { return max(max(a, b), c); }
// 16-byte global -> shared copy that bypasses the registers (completes at cp_async_wait_all)
__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// a padding block of a stored row (poa_types.h: DpState): the out-of-band values H = inf_min, D = 0, so that every sector the
// warp writes is whole. tp: the block's chunk 0, cs: ints between chunks
__device__ __forceinline__ void store_pad(int *tp, int64_t cs, int NEG) {
#pragma unroll
    for (int c = 0; c < TB / CHUNK; ++c) st4(tp + c * cs, c < CPT / CHUNK ? NEG : 0, c < CPT / CHUNK ? NEG : 0, c < CPT / CHUNK ? NEG : 0, c < CPT / CHUNK ? NEG : 0);
}


// ---- the two per-thread passes over a row's 16 cells, in a branch-free form -------------------------------------
// The block scan of the F states runs in "A space": A1'[k] = H'[k] + k*e1 (the constant -o1 is applied when F is read back),
// so F1[j] = max_{k<j} A1'[k] - o1 - j*e1 and the scan identity is inf_min + beg*e1 + o1. Within a thread neither pass forms
// the per-column offsets k*e: pass 1 folds its cells' A values right to left (Horner), pass 2 runs the F recurrence itself.
// MASKED = some of the thread's columns lie outside [beg, end] (they must come out as exactly inf_min).
//
// mbase: shared-memory address of smat (256-byte aligned, so its low byte is 0); qo: byte k of word c is
// 32 * (the row's graph base) + 4 * (query code of my column 4c + k), the low byte of that column's entry address
template <bool MASKED>
__device__ __forceinline__ void row_pass1(int (&H)[CPT], int (&E1)[CPT], int (&E2)[CPT], unsigned mbase, const uint32_t (&qo)[4],
                                          int j0, int beg, int end, int NEG, int e1, int e2, int &agg1, int &agg2) {
#pragma unroll
    for (int e = 0; e < CPT; ++e) {
        const int s = lds_const(__byte_perm(qo[e >> 2], mbase, 0x7650 | (e & 3)));   // the entry's address, one PRMT
        int h = __vimax3_s32(H[e] + s, E1[e], E2[e]);                    // H' = max(M + s, E1, E2), :1033,1050
        if (MASKED) {
            const bool inb = (unsigned)(j0 + e - beg) <= (unsigned)(end - beg);
            h = inb ? h : NEG; E1[e] = inb ? E1[e] : NEG; E2[e] = inb ? E2[e] : NEG;
        }
        H[e] = h;
    }
    // a = max_k H'[k] + k*e over my cells, folded right to left: a <- max(a + e, H'[k]); then the thread's aggregate in A space
    int a1 = H[CPT - 1], a2 = H[CPT - 1];
#pragma unroll
    for (int e = CPT - 2; e >= 0; --e) { a1 = __viaddmax_s32(a1, e1, H[e]); a2 = __viaddmax_s32(a2, e2, H[e]); }
    agg1 = max(agg1, a1 + j0 * e1); agg2 = max(agg2, a2 + j0 * e2);
}

// folds chunk oc of a predecessor row (4 H values, 4 D codes) into my columns' candidates: H[e+1] <- the M input H_pred[e],
// E1 / E2 <- max with the decoded E values. ROW0: the predecessor may be row 0, whose D holds the E_NEG16 sentinel (every
// other row's codes lie in [e, oe], poa_types.h: DpState)
template <bool ROW0>
__device__ __forceinline__ void pred_chunk(int (&H)[CPT], int (&E1)[CPT], int (&E2)[CPT], int oc, int4 h4, int4 d4, int NEG) {
    const int h[CHUNK] = {h4.x, h4.y, h4.z, h4.w}, dv[CHUNK] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
    for (int u = 0; u < CHUNK; ++u) {
        const int e = oc * CHUNK + u;
        const int c1 = dv[u] & 0xffff, c2 = (int)((unsigned)dv[u] >> 16);
        if (e + 1 < CPT) H[e + 1] = max(H[e + 1], h[u]);
        E1[e] = max(E1[e], ROW0 && c1 == E_NEG16 ? NEG : h[u] - c1); E2[e] = max(E2[e], ROW0 && c2 == E_NEG16 ? NEG : h[u] - c2);
    }
}

// MODE 0: all of the warp's active columns are inside the band; 1: some lie left (or left and right) of it -- every value
// of an outside cell is forced to inf_min; 2: some lie right of it only -- nothing in the band depends on those cells
// and the traceback never reads the F planes outside the band, so only H / E1 / E2 are forced (they feed later rows).
// RING_NT: threads per CTA if the row also goes to the shared-memory ring (rs: address of my chunk 0 of the slot), else 0.
// F1 / F2: the insertion states of my first column, P - o - j0*e from the block scan's exclusive prefix P. From there the
// recurrence F[j+1] = max(F[j] - e, H'[j] - oe) gives, integer for integer, the A-space value max_{k<=j} A'[k] - o - (j+1)*e
// (both sides are max(P, max_{k<=j} H'[k] + k*e) - o - (j+1)*e), so the pass forms no F value the A-space scan does not; the
// other terms, F - e and H' - oe, lie at most oe below an F value or an H' value, as h - oe of the E update does. The int32 range
// argument of the A-space sweep (DESIGN section 7: nothing above H' + (j+1)*e) therefore covers this pass unchanged.
template <int MODE, int RING_NT>
__device__ __forceinline__ void row_pass2(int (&H)[CPT], int (&E1)[CPT], int (&E2)[CPT], int F1, int F2, int j0, int beg, int end, int NEG,
                                          int e1, int e2, int oe1, int oe2, int *tp, int64_t cs, unsigned rs, int &tmax) {
    // one H chunk and one D chunk per 4 cells (tp: the thread's chunk 0, cs: ints between chunks; poa_types.h: DpState)
#pragma unroll
    for (int oc = 0; oc < CPT / CHUNK; ++oc) {
        int dd[CHUNK];
#pragma unroll
        for (int u = 0; u < CHUNK; ++u) {
            const int e = oc * CHUNK + u, hp = H[e];                       // H' of the cell, before F
            int h = __vimax3_s32(hp, F1, F2);                              // :1067 (F used, not stored)
            F1 = __viaddmax_s32(F1, -e1, hp - oe1); F2 = __viaddmax_s32(F2, -e2, hp - oe2);   // F of the next column
            int x1 = __viaddmax_s32(E1[e], -e1, h - oe1);                  // E for the next rows, :1070-1071
            int x2 = __viaddmax_s32(E2[e], -e2, h - oe2);
            if (MODE == 1) {
                const bool inb = (unsigned)(j0 + e - beg) <= (unsigned)(end - beg);
                h = inb ? h : NEG; x1 = inb ? x1 : NEG; x2 = inb ? x2 : NEG;
            } else if (MODE == 2) {
                const bool inb = j0 + e <= end;
                h = inb ? h : NEG; x1 = inb ? x1 : NEG; x2 = inb ? x2 : NEG;
            }
            H[e] = h; E1[e] = x1; E2[e] = x2;
            dd[u] = __byte_perm(h - x1, h - x2, 0x5410);                  // (h-x1) | (h-x2) << 16: e <= H - E' <= oe < 65535 (0 outside the band)
            tmax = max(tmax, h);
        }
        st4(tp + oc * cs, H[oc * CHUNK], H[oc * CHUNK + 1], H[oc * CHUNK + 2], H[oc * CHUNK + 3]);
        st4(tp + (CPT / CHUNK + oc) * cs, dd[0], dd[1], dd[2], dd[3]);
        if (RING_NT) {
            sts4(rs + oc * RING_NT * 16, H[oc * CHUNK], H[oc * CHUNK + 1], H[oc * CHUNK + 2], H[oc * CHUNK + 3]);
            sts4(rs + (CPT / CHUNK + oc) * RING_NT * 16, dd[0], dd[1], dd[2], dd[3]);
        }
    }
}

// left/right-most column of the thread's cells that attain v (only in-band cells count)
template <bool MASKED>
__device__ __forceinline__ void row_argmax(const int (&H)[CPT], int v, int j0, int beg, int end, int &tl, int &tr) {
    unsigned m = 0;
#pragma unroll
    for (int e = 0; e < CPT; ++e) m |= H[e] == v ? 1u << e : 0u;
    if (MASKED) {
        const int lo = max(beg - j0, 0), hi = min(end - j0, CPT - 1);
        m &= (2u << hi) - (1u << lo);
    }
    if (m) { tl = j0 + __ffs(m) - 1; tr = j0 + 31 - __clz(m); }
}

// ---------------------------------------------------------------------------------------------------------
// banded convex-gap DP of query q[1..L] against the sorted graph. All threads of the CTA; L + 1 <= 16 * blockDim.x.
// Returns the number of banded cells (sum of dp_end-dp_beg+1), or -1 if the planes outgrew the slot.
//
// The ring: where the class's dynamic shared memory holds two rows (every class but t1024), each row also goes to slot
// r & 1 of a ring there, chunk-major like the planes but with a block for every thread of the CTA: chunk c of thread t at
// int (c * NT + t) * CHUNK of the slot, so a warp's access to a chunk is 512 contiguous bytes. ring_info[r & 1] holds the
// row's band. A predecessor at r - 2 is read from there instead of from L2. No extra barrier guards the slots: row r reads
// slot r & 1 (row r - 2) before its first barrier and overwrites it only in its second pass, after that barrier; tid 0 writes
// ring_info[r & 1] after the second barrier, and row r + 1, which reads the other slot, starts after both. Rows r - 1 and
// r - 2 wrote their slots before barriers row r has already passed.
// ---------------------------------------------------------------------------------------------------------
template <int NT>
__device__ long long dp_sweep(KShared &S, const BatchArgs &A, const uint8_t *__restrict__ qg, int L, uint4 *qsm, unsigned ring) {
    constexpr int RING_NT = poa_ring_bytes(NT) ? NT : 0;                        // a compile-time property of the class
    constexpr unsigned SLOT = NT * TB * sizeof(int), RCS = NT * 16;              // ring bytes per slot, between chunks
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = NT >> 5;
    const unsigned my_ring = ring + tid * 16;                                       // my chunk 0 of slot 0
    const PoaParams &P = A.P;
    // slot arrays addressed from the kernel parameters (not through the pointers cached in shared memory), so that the
    // compiler knows they are global memory and emits LDG/STG instead of generic accesses
    uint8_t *const sb = A.slots + (int64_t)blockIdx.x * A.lay.slot_bytes;
    const RowRec *const rec_tab = reinterpret_cast<const RowRec *>(sb + A.lay.o_row_rec);
    const int *const pre_row = reinterpret_cast<const int *>(sb + A.lay.o_pre_row);
    RowInfo *const info = reinterpret_cast<RowInfo *>(sb + A.lay.o_row_info);
    int64_t *const row_off = reinterpret_cast<int64_t *>(sb + A.lay.o_row_off);
    int *const planes = A.planes + (int64_t)blockIdx.x * A.lay.plane_cap;
    const int64_t plane_cap = A.lay.plane_cap;
    const int node_n = S.g.node_n, R = node_n - 1;
    const int NEG = P.inf_min, e1 = P.e1, e2 = P.e2, oe1 = P.o1 + P.e1, oe2 = P.o2 + P.e2;
    const int w = P.wb + (int)(P.wf * L);                                    // abpoa_align_simd.c:474
    const int pn_shift = reference_lane_count(P, L, node_n) == 16 ? 4 : 3;
    static_assert(CPT == 16, "shifts below assume 16 columns per thread");
    const int j0 = tid * CPT;

    // query codes of my 16 columns as byte offsets 4 * code into a row of smat, one byte each (column j scores against
    // q_j = qg[j-1]; column 0 and columns past the query score 0, abpoa_align_simd.c:536). A row adds 32 * base to every
    // byte: 32 * 4 + 4 * 5 < 256, no byte carries into the next
    uint32_t qo[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int e = 0; e < CPT; ++e) {
        const int j = j0 + e;
        const uint32_t c = (j >= 1 && j <= L) ? qg[j - 1] : 5u;
        qo[e >> 2] |= (4u * c) << ((e & 3) * 8);
    }
    // they are read back from shared memory in every row (only by this thread, one 128-bit load): codes kept in registers across
    // the row loop let the compiler hoist 16 per-column table offsets out of it, which then spilled
    qsm[tid] = make_uint4(qo[0], qo[1], qo[2], qo[3]);
    const unsigned smat_s = (unsigned)__cvta_generic_to_shared(S.smat);           // low byte 0 (256-byte aligned)

    int H[CPT], E1[CPT], E2[CPT];          // the previous row's values of my columns (valid iff prev_active)
    bool prev_active;
    int prev_beg = 0, prev_end, prev_left = 0, prev_right = 0;
    int cur_blk = 0, cells = 0;               // row blocks (of TB ints) written so far; banded cells so far

    // ---- row 0 (simd_abpoa_cg_first_dp, :617-688) ----
    {
        const int dd = L - rec_tab[0].rd;
        prev_end = min(L, max(0, dd) + w);
        const int nT = prev_end / CPT + 1, nTs = row_blocks(0, prev_end);
        if ((int64_t)nTs * TB > plane_cap) return -1;
        prev_active = tid < nT;
        // the threads past the band (the padding block among them) hold out-of-band values
        int D[CPT];
#pragma unroll
        for (int e = 0; e < CPT; ++e) {
            const int j = j0 + e;
            if (j == 0) { H[e] = 0; E1[e] = -oe1; E2[e] = -oe2; D[e] = oe1 | (oe2 << 16); }
            else if (j <= prev_end) { H[e] = max(-P.o1 - e1 * j, -P.o2 - e2 * j); E1[e] = NEG; E2[e] = NEG; D[e] = E_NEG16 | (E_NEG16 << 16); }
            else { H[e] = E1[e] = E2[e] = NEG; D[e] = 0; }
        }
        if (tid < nTs) {
            int *tp = planes + chunk_index(nTs, tid, 0);
            const int64_t cs = chunk_index(nTs, 0, 1);
#pragma unroll
            for (int oc = 0; oc < CPT / CHUNK; ++oc) {
                st4(tp + oc * cs, H[oc * CHUNK], H[oc * CHUNK + 1], H[oc * CHUNK + 2], H[oc * CHUNK + 3]);
                st4(tp + (CPT / CHUNK + oc) * cs, D[oc * CHUNK], D[oc * CHUNK + 1], D[oc * CHUNK + 2], D[oc * CHUNK + 3]);
            }
        }
        if (RING_NT) {
#pragma unroll
            for (int oc = 0; oc < CPT / CHUNK; ++oc) {
                sts4(my_ring + oc * RCS, H[oc * CHUNK], H[oc * CHUNK + 1], H[oc * CHUNK + 2], H[oc * CHUNK + 3]);
                sts4(my_ring + (CPT / CHUNK + oc) * RCS, D[oc * CHUNK], D[oc * CHUNK + 1], D[oc * CHUNK + 2], D[oc * CHUNK + 3]);
            }
        }
        if (lane == 31) S.wM[0][3][warp] = H[CPT - 1];
        if (tid == 0) {
            RowInfo ri; ri.beg = 0; ri.end = prev_end; ri.left = 0; ri.right = 0; info[0] = ri; row_off[0] = 0;
            if (RING_NT) S.ring_info[0] = ri;
        }
        cur_blk = nTs; cells = prev_end + 1;
        if (tid == 0) { cp_async16(&S.rec[1], rec_tab + (R > 1 ? 1 : 0)); cp_async_wait_all(); }
    }
    __syncthreads();

    for (int r = 1; r < R; ++r) {
        const int par = r & 1;
        const RowRec rec = S.rec[par];
        // the next row's record, in flight while this row computes (its buffer was last read two barriers ago)
        if (tid == 0 && r + 1 < R) cp_async16(&S.rec[par ^ 1], rec_tab + r + 1);
        // ---- band of the row (GET_AD_DP_BEGIN/END + lane-group snap, :946-960) ----
        const int b = rec.base_npre & 0xff, npre = rec.base_npre >> 8;
        const int dd = L - rec.rd;
        int maxL = node_n, maxR = 0, min_pre_beg = 0x7fffffff;
        bool has_prev = false;
        if (npre == 1 && rec.pre0 == r - 1) {                       // the linear-chain case: everything is in registers
            maxL = min(node_n, prev_left + 1); maxR = prev_right + 1; min_pre_beg = prev_beg; has_prev = true;   // max_pos_left starts at node_n (abpoa_graph.c:347-352)
        } else {
#pragma unroll 1
            for (int k = 0; k < npre; ++k) {
                const int p = k == 0 ? rec.pre0 : pre_row[rec.pre_off + k];
                int pl, pr, pb;
                if (p == r - 1) { pl = prev_left; pr = prev_right; pb = prev_beg; has_prev = true; }
                else if (RING_NT && p == r - 2) { const RowInfo pi = S.ring_info[par]; pl = pi.left; pr = pi.right; pb = pi.beg; }
                else { const RowInfo pi = info[p]; pl = pi.left; pr = pi.right; pb = pi.beg; }
                maxL = min(maxL, pl + 1); maxR = max(maxR, pr + 1); min_pre_beg = min(min_pre_beg, pb);
            }
        }
        const bool only_prev = npre == 1 && has_prev;
        int beg = max(0, min(maxL, dd) - w);
        const int end = min(L, max(maxR, dd) + w);
        if ((beg >> pn_shift) < (min_pre_beg >> pn_shift)) beg = min_pre_beg;
        const int t0 = beg >> 4, nT = (end >> 4) - t0 + 1, tt = tid - t0;
        const int nTs = row_blocks(beg, end), tts = tid - row_t0(beg);   // stored blocks, my stored block (poa_types.h: DpState)
        if ((int64_t)(cur_blk + nTs) * TB > plane_cap) return -1;       // uniform across the CTA
        const bool active = tt >= 0 && tt < nT;
        // masking is decided per WARP (no divergent double execution): 0 = all active threads inside the band,
        // 1 = some columns left of the band, 2 = some columns right of it only
        const int wmode = __any_sync(FULL, active && j0 < beg) ? 1 : __any_sync(FULL, active && j0 + CPT - 1 > end) ? 2 : 0;
        const uint32_t qadd = 0x01010101u * (32u * b);                  // table row b: 32 * b added to every byte offset

        // H of the column left of my first one, previous row
        int hl = __shfl_up_sync(FULL, prev_active ? H[CPT - 1] : NEG, 1);
        if (lane == 0) hl = warp > 0 ? S.wM[par ^ 1][3][warp - 1] : NEG;

        const int id1 = NEG + beg * e1 + P.o1, id2 = NEG + beg * e2 + P.o2;   // identities of the two scans ("A space")
        int agg1 = id1, agg2 = id2;
        if (active) {
            // M candidates: H[e] <- H_pred[e-1]; E candidates stay in E1/E2 (previous row = predecessor case)
            if (has_prev && prev_active) {
#pragma unroll
                for (int e = CPT - 1; e >= 1; --e) H[e] = H[e - 1];
                H[0] = hl;
            } else {
#pragma unroll
                for (int e = 0; e < CPT; ++e) { H[e] = NEG; E1[e] = NEG; E2[e] = NEG; }
                if (has_prev) H[0] = hl;
            }
            // predecessors further back: row r - 2 from the ring, older ones from the planes in global memory
#pragma unroll 1
            for (int k = only_prev ? npre : 0; k < npre; ++k) {
                const int p = k == 0 ? rec.pre0 : pre_row[rec.pre_off + k];
                if (p == r - 1) continue;
                if (RING_NT && p == r - 2) {
                    const RowInfo pi = S.ring_info[par];
                    const int pt0 = pi.beg >> 4, pnT = (pi.end >> 4) - pt0 + 1, ptt = tid - pt0;
                    const unsigned rs = my_ring + par * SLOT;
                    if (ptt >= 0 && ptt < pnT) {
                        if (p == 0) {                                             // uniform across the CTA
#pragma unroll
                            for (int oc = 0; oc < CPT / CHUNK; ++oc) pred_chunk<true>(H, E1, E2, oc, lds4(rs + oc * RCS), lds4(rs + (CPT / CHUNK + oc) * RCS), NEG);
                        } else {
#pragma unroll
                            for (int oc = 0; oc < CPT / CHUNK; ++oc) pred_chunk<false>(H, E1, E2, oc, lds4(rs + oc * RCS), lds4(rs + (CPT / CHUNK + oc) * RCS), NEG);
                        }
                    }
                    // H[16*tid - 1]: the last H (chunk 3) of the left neighbour's block
                    if (ptt >= 1 && ptt <= pnT) H[0] = max(H[0], lds1(rs + (CPT / CHUNK - 1) * RCS - 4));
                    continue;
                }
                const RowInfo pi = info[p];
                const int pt0 = pi.beg >> 4, pnT = (pi.end >> 4) - pt0 + 1, ptt = tid - pt0, pnTs = row_blocks(pi.beg, pi.end);
                const int *Hp = planes + row_off[p] + chunk_index(pnTs, tid - row_t0(pi.beg), 0);   // my block of row p (if stored)
                const int64_t pcs = chunk_index(pnTs, 0, 1);
                if (ptt >= 0 && ptt < pnT) {
#pragma unroll
                    for (int oc = 0; oc < CPT / CHUNK; ++oc) pred_chunk<true>(H, E1, E2, oc, ld4cg(Hp + oc * pcs), ld4cg(Hp + (CPT / CHUNK + oc) * pcs), NEG);
                }
                // H[16*tid - 1]: the last H (chunk 3) of the left neighbour's block
                if (ptt >= 1 && ptt <= pnT) H[0] = max(H[0], __ldcg(Hp - CHUNK + (CPT / CHUNK - 1) * pcs + CHUNK - 1));
            }
            const uint4 q4 = qsm[tid];
            const uint32_t qo[4] = {q4.x + qadd, q4.y + qadd, q4.z + qadd, q4.w + qadd};
            if (wmode != 1) row_pass1<false>(H, E1, E2, smat_s, qo, j0, beg, end, NEG, e1, e2, agg1, agg2);
            else row_pass1<true>(H, E1, E2, smat_s, qo, j0, beg, end, NEG, e1, e2, agg1, agg2);
        }
        // ---- exclusive prefix maximum over the row: warp shuffle scan + redux over warp aggregates ----
        int inc1 = agg1, inc2 = agg2;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int n1 = __shfl_up_sync(FULL, inc1, off), n2 = __shfl_up_sync(FULL, inc2, off);
            if (lane >= off) { inc1 = max(inc1, n1); inc2 = max(inc2, n2); }
        }
        int ex1 = __shfl_up_sync(FULL, inc1, 1), ex2 = __shfl_up_sync(FULL, inc2, 1);
        if (lane == 0) { ex1 = id1; ex2 = id2; }
        if (lane == 31) { S.wF[par][0][warp] = inc1; S.wF[par][1][warp] = inc2; }
        __syncthreads();
        int P1, P2;
        {
            const int wv1 = lane < warp ? S.wF[par][0][lane] : id1, wv2 = lane < warp ? S.wF[par][1][lane] : id2;
            P1 = max(__reduce_max_sync(FULL, wv1), ex1); P2 = max(__reduce_max_sync(FULL, wv2), ex2);
        }
        // the row maximum starts below every value a cell can hold. Not inf_min minus a constant: inf_min lies only
        // max(min_mis, o1 + e1, o2 + e2) + 512 * max(e1, e2) above INT32_MIN, which wraps for extensions of at most 1. The reference
        // counts only cells above inf_min (simd_abpoa_max_in_row); every row a band reaches has one (a predecessor's argmax column or
        // the one right of it), so both find the same maximum
        int tmax = INT32_MIN;
        {
            int *tp = planes + (int64_t)cur_blk * TB + chunk_index(nTs, tts, 0);
            const int64_t cs = chunk_index(nTs, 0, 1);
            const unsigned rs = my_ring + par * SLOT;
            if (active) {
                const int F1 = P1 - P.o1 - j0 * e1, F2 = P2 - P.o2 - j0 * e2;   // F of my first column
                if (wmode == 0) row_pass2<0, RING_NT>(H, E1, E2, F1, F2, j0, beg, end, NEG, e1, e2, oe1, oe2, tp, cs, rs, tmax);
                else if (wmode == 2) row_pass2<2, RING_NT>(H, E1, E2, F1, F2, j0, beg, end, NEG, e1, e2, oe1, oe2, tp, cs, rs, tmax);
                else row_pass2<1, RING_NT>(H, E1, E2, F1, F2, j0, beg, end, NEG, e1, e2, oe1, oe2, tp, cs, rs, tmax);
            } else if ((unsigned)tts < (unsigned)nTs) store_pad(tp, cs, NEG);
        }
        // ---- left/right-most argmax of H over the band (simd_abpoa_max_in_row, :1107-1119) ----
        {
            const int wmax = __reduce_max_sync(FULL, tmax);
            int tleft = 0x7fffffff, tright = -1;
            if (active && tmax == wmax) {
                if (wmode == 0) row_argmax<false>(H, wmax, j0, beg, end, tleft, tright); else row_argmax<true>(H, wmax, j0, beg, end, tleft, tright);
            }
            const int wl = __reduce_min_sync(FULL, tleft), wr = __reduce_max_sync(FULL, tright);
            if (lane == 0) { S.wM[par][0][warp] = wmax; S.wM[par][1][warp] = wl; S.wM[par][2][warp] = wr; }
            if (lane == 31) S.wM[par][3][warp] = active ? H[CPT - 1] : NEG;
        }
        if (tid == 0) cp_async_wait_all();
        __syncthreads();
        {
            const int v = lane < nwarps ? S.wM[par][0][lane] : INT32_MIN;       // lanes without a warp: below every maximum
            const int bmax = __reduce_max_sync(FULL, v);
            const int l = (lane < nwarps && v == bmax) ? S.wM[par][1][lane] : 0x7fffffff;
            const int rr = (lane < nwarps && v == bmax) ? S.wM[par][2][lane] : -1;
            prev_left = __reduce_min_sync(FULL, l); prev_right = __reduce_max_sync(FULL, rr);
        }
        prev_beg = beg; prev_end = end; prev_active = active;
        if (tid == 0) {
            RowInfo ri; ri.beg = beg; ri.end = end; ri.left = prev_left; ri.right = prev_right; info[r] = ri; row_off[r] = (int64_t)cur_blk * TB;
            if (RING_NT) S.ring_info[par] = ri;
        }
        cur_blk += nTs; cells += end - beg + 1;
    }
    __syncthreads();
    return cells;
}

#define PHASE_TICK(ph) do { if (A.phase_clk && threadIdx.x == 0) { unsigned long long _n = clock64(); A.phase_clk[(size_t)blockIdx.x * PH_N + (ph)] += _n - t_last; t_last = _n; } } while (0)

template <int NT>
__device__ __forceinline__ void poa_msa_body(const BatchArgs &A) {
    extern __shared__ __align__(16) unsigned char dyn_smem[];    // scratch of the topological sort (poa_cta.cuh), the sweep's row ring
    __shared__ KShared S;
    __shared__ uint4 qsm[NT];                                    // query codes of each thread's columns (dp_sweep)
    const int tid = threadIdx.x;
    int *ws = &S.wF[0][0][0];
    // the slot index as an int: addresses formed exactly as dp_sweep forms its own (from the unsigned blockIdx.x) would be
    // computed once here and kept live through the whole kernel, which spills t64 .. t256
    if (tid == 0) { const int slot = blockIdx.x; slot_views(A.lay, A.slots + (int64_t)slot * A.lay.slot_bytes, A.planes + (int64_t)slot * A.lay.plane_cap, S.g, S.rt, S.d); }
    for (int k = tid; k < 40; k += blockDim.x) S.smat[k] = (k & 7) < 5 ? A.P.mat[(k >> 3) * 5 + (k & 7)] : 0;
    unsigned long long t_last = A.phase_clk ? clock64() : 0ULL, t_start = t_last;
    __syncthreads();

    while (true) {
        if (tid == 0) {
            const int k = atomicAdd(A.next_job, 1);
            int j = -1;
            if (k < A.n_jobs) j = A.job_base + k;
            S.job = j;
        }
        __syncthreads();
        const int job = S.job;
        if (job < 0) break;
        const JobDesc jd = A.jobs[job];
        const int K = jd.n_seq;
        const int *lens = A.lens + jd.len_off;
        const int64_t *soff = A.soff + jd.len_off;
        const uint8_t *seqs = A.seqs + jd.seq_off;
        if (tid == 0) { graph_reset(S.g, K); S.abort_s = 0; }
        __syncthreads();
        // read order: the job's guide tree (abpoa_seed.c:705-722), computed by guide_tree_kernel before this launch (guide_tree.cu)
        const int *const order = A.order + jd.len_off;
        if (tid == 0 && A.gt_status[job]) S.g.err = JOB_ERR_GT_CAP;
        __syncthreads();
        long long cells = 0;
        for (int a = 0; a < K && !S.g.err; ++a) {
            const int read = order[a], L = lens[read];
            const uint8_t *q = seqs + soff[read];
            if (a == 0) {
                if (A.serial_phases) { if (tid == 0) graph_add_first_sequence(S.g, q, L, read); }
                else cta_add_first_sequence(S.g, q, L, read);
                PHASE_TICK(PH_FUSE);
            } else {
                long long c = -2;
                if (L + 1 <= CPT * (int)blockDim.x) c = dp_sweep<NT>(S, A, q, L, qsm, (unsigned)__cvta_generic_to_shared(dyn_smem));
                if (c < 0) { if (tid == 0) S.g.err = c == -2 ? JOB_ERR_QUERY_LEN : JOB_ERR_PLANE_CAP; c = 0; }
                cells += c;
                __syncthreads();
                PHASE_TICK(PH_DP);
                if (A.serial_phases) { if (tid == 0 && !S.g.err) { dp_best_cell(S.g, S.rt, S.d, A.P, L); dp_backtrack(S.g, S.rt, S.d, A.P, q, L); } }
                else if (tid < 32 && !S.g.err) warp_backtrack(S.g, S.rt, S.d, A.P, S.smat, q, L);
                PHASE_TICK(PH_BACKTRACK);
                __syncthreads();
                if (A.serial_phases) { if (tid == 0 && !S.g.err) graph_fuse_alignment(S.g, q, S.d.cigar, S.d.n_cigar, read); }
                else if (!S.g.err) cta_fuse_alignment(S.g, q, L, S.d.cigar, S.d.n_cigar, read, ws);
                PHASE_TICK(PH_FUSE);
            }
            __syncthreads();
            if (S.g.err) break;
            if (A.serial_phases) { if (tid == 0) graph_topo_sort_serial(S.g, S.rt); __syncthreads(); }
            else cta_topo_sort(S.g, S.rt, dyn_smem, A.scratch_bytes, ws, A.bfs_order == 0);
            PHASE_TICK(PH_TOPO);
            if (S.g.err) break;
        }
        __syncthreads();
        // ---- MSA (abpoa_generate_rc_msa, abpoa_output.c:149-176) ----
        if (!S.g.err) {
            if (A.serial_phases) { if (tid == 0) S.msa_len_s = graph_msa_rank(S.g); __syncthreads(); }
            else cta_msa_rank(S.g, dyn_smem, A.scratch_bytes, ws, &S.msa_len_s);
            if (tid == 0 && !S.g.err && S.msa_len_s > jd.msa_stride) S.g.err = JOB_ERR_MSA_CAP;
        }
        __syncthreads();
        if (!S.g.err) {
            const int ml = S.msa_len_s;
            uint8_t *msa = A.msa + jd.msa_off;
            for (int64_t i = tid; i < (int64_t)K * ml; i += blockDim.x) msa[(i / ml) * jd.msa_stride + (i % ml)] = GAP_CODE;
            __syncthreads();
            for (int v = 2 + tid; v < S.g.node_n; v += blockDim.x) graph_msa_fill_node(S.g, v, msa, jd.msa_stride);
        }
        __syncthreads();
        if (tid == 0) { A.status[job] = S.g.err; A.msa_len[job] = S.g.err ? 0 : S.msa_len_s; A.cells[job] = cells; }
        PHASE_TICK(PH_MSA);
        __syncthreads();
    }
    if (A.phase_clk && tid == 0) A.phase_clk[(size_t)blockIdx.x * PH_N + PH_TOTAL] += clock64() - t_start;
}

// One entry point per CTA-size class (the register budget per thread follows from the launch bounds):
//   queries up to 511 bases -> one warp, 16 CTAs per SM;  up to 1023 -> 64 threads;
//   up to 2047 -> 128 threads, 4 CTAs per SM;  up to 4095 -> 256 threads, 2 per SM;
//   up to 10239 (covers Cactus' 10 kbp window) -> 640 threads;  up to 16383 -> 1024 threads.
extern "C" __global__ void __launch_bounds__(32, 16) poa_msa_kernel_t32(const BatchArgs A) { poa_msa_body<32>(A); }
extern "C" __global__ void __launch_bounds__(64, 8) poa_msa_kernel_t64(const BatchArgs A) { poa_msa_body<64>(A); }
#ifndef BARB200_T128_MINB
#define BARB200_T128_MINB 4
#endif
extern "C" __global__ void __launch_bounds__(128, BARB200_T128_MINB) poa_msa_kernel_t128(const BatchArgs A) { poa_msa_body<128>(A); }
extern "C" __global__ void __launch_bounds__(256, 2) poa_msa_kernel_t256(const BatchArgs A) { poa_msa_body<256>(A); }
extern "C" __global__ void __launch_bounds__(640, 1) poa_msa_kernel_t640(const BatchArgs A) { poa_msa_body<640>(A); }
extern "C" __global__ void __launch_bounds__(1024, 1) poa_msa_kernel_t1024(const BatchArgs A) { poa_msa_body<1024>(A); }

}  // namespace barb200
