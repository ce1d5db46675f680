/*
 * barb200.h -- C ABI of libbarb200.so, the H100-native engine behind Cactus' base-alignment-refinement (BAR)
 * phase: POA mode (abPOA's partial-order alignments, below) and cPecan mode (the banded pair-HMM posteriors, further
 * down: barb200_pecan_*). Plain pointers and sizes only; no CUDA, torch or C++ types cross this boundary.
 *
 * Drop-in boundary (paths relative to the Cactus source tree, commit 2a4a172f):
 *   - barb200_poa_msa_batch ........ replaces the abpoa_init / abpoa_msa / abpoa_free triple the shim issues once per
 *                                    sliding window of every end (bar/impl/poaBarAligner.c:565-628;
 *                                    submodules/abPOA/include/abpoa.h:150-160), for MANY windows at once.
 *   - barb200_msa_make_partial_order_alignment[_batch]
 *                                    replaces msa_make_partial_order_alignment (bar/inc/poaBarAligner.h:76,
 *                                    bar/impl/poaBarAligner.c:463-749): windows, overlap trimming, stitching.
 *   - barb200_make_consistent_partial_order_alignments
 *                                    replaces make_consistent_partial_order_alignments (bar/inc/poaBarAligner.h:108,
 *                                    bar/impl/poaBarAligner.c:751-801): all ends of a flower in one batched launch,
 *                                    then the serial cross-end trimming.
 *   - barb200_params ............... the fields abpoaParamaters_constructFromCactusParams reads from the <bar><poa>
 *                                    XML element (bar/impl/poaBarAligner.c:24-81; keys listed in
 *                                    src/cactus/cactus_progressive_config.xml:307-325).
 * INTEGRATION.md shows the ~40-line C shim that re-exports the reference symbols on top of these.
 *
 * Error convention: functions return 0 on success and a negative BARB200_E* code on failure;
 * barb200_last_error() gives the message. (The reference aborts the process instead, st_errAbort /
 * err_fatal; the shim in INTEGRATION.md converts a non-zero return into st_errAbort to keep that behaviour.)
 * There is NO CPU fallback: without a CUDA device barb200_create fails.
 *
 * Thread safety: a context may be shared by threads (the reference calls msa_make_partial_order_alignment concurrently from
 * OpenMP teams, bar/impl/bar.c:90-94). The MSA-level calls below go through one queue of ends per context: whatever several
 * threads have submitted when a device lane becomes free runs as ONE device batch; barb200_flower_submit / _wait expose the
 * queue directly so that a caller can submit every end of every leaf flower before waiting for the first (SURVEY.md 8b / 8(f)-2).
 */
#ifndef BARB200_H
#define BARB200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BARB200_OK 0
#define BARB200_ENODEV (-1)     /* no usable CUDA device / driver */
#define BARB200_ENOMEM (-2)     /* device or host allocation failed */
#define BARB200_EINVAL (-3)     /* bad argument (empty sequence, code > 4, gap model other than convex, ...) */
#define BARB200_ECUDA (-4)      /* a CUDA call or the kernel failed */
#define BARB200_EJOB (-5)       /* a job failed on the device (graph error the reference would abort on) */

typedef struct barb200_ctx barb200_ctx;

typedef struct {
    /* scoring and banding -- bar/impl/poaBarAligner.c:36-77 */
    int mat[25];                 /* partialOrderAlignmentSubMatrix, 5x5 ACGTN */
    int gap_open1, gap_ext1;     /* partialOrderAlignmentGapOpenPenalty1 / GapExtensionPenalty1 */
    int gap_open2, gap_ext2;     /* partialOrderAlignmentGapOpenPenalty2 / GapExtensionPenalty2 (convex: both opens > 0) */
    int wb; float wf;            /* partialOrderAlignmentBandConstant / BandFraction; band = wb + wf*len */
    /* guide tree -- bar/impl/poaBarAligner.c:46-53 */
    int k, w, min_w;             /* partialOrderAlignmentMinimizerK / W / MinW */
    int progressive_poa;         /* partialOrderAlignmentProgressiveMode */
    int disable_seeding;         /* partialOrderAlignmentDisableSeeding; must be 1 (Cactus' default) */
    /* engine */
    int device;                  /* CUDA device ordinal */
    int threads_per_block;       /* 0 = auto: every job runs in the smallest CTA class (32..1024 threads) its longest sequence fits; > 0: minimum class */
    int ctas_per_sm;             /* 0 = auto (occupancy / memory limited) */
    double mem_fraction;         /* fraction of free device memory the slots may take; 0 = 0.85 */
    int host_threads;            /* threads for host-side packing / guide trees; 0 = all */
    int collect_phase_clocks;    /* 1: accumulate per-phase SM clock counters (profiling aid) */
    /* several GPUs behind ONE context (cactus_consolidated is one process): n_devices > 0 -> devices[0 .. n_devices),
     * n_devices < 0 -> every visible device, 0 -> the single `device` above. Ends are dealt to the devices by estimated cost
     * (batch call) or pulled by whichever device lane is free (end queue); results land in the caller's buffers. */
    int n_devices;
    int devices[8];
    int lanes;                   /* batches in flight per device, 1 or 2; 0 = 2 */
} barb200_params;

/* Cactus' defaults (src/cactus/cactus_progressive_config.xml:307-325) */
void barb200_params_default(barb200_params *p);

barb200_ctx *barb200_create(const barb200_params *p, char *errbuf, int errbuf_len);
void barb200_destroy(barb200_ctx *ctx);
const char *barb200_last_error(barb200_ctx *ctx);

/* One job = one abpoa_msa call: n_seq[i] sequences of codes 0..4 (A,C,G,T,N), concatenated over all jobs in
 * `seqs` with lengths in `seq_lens` (sum of n_seq entries). progressive[i] (may be NULL = use params) is the
 * per-job abpt->progressive_poa the shim decides at poaBarAligner.c:567-571.
 * Outputs: msa_out[i] = malloc'd n_seq[i] x msa_len[i] row-major bytes (0-3 ACGT, 4 N, 5 gap), to be released
 * with barb200_free; cells[i] (may be NULL) = banded DP cells of the job (sum of dp_end-dp_beg+1). */
int barb200_poa_msa_batch(barb200_ctx *ctx, int64_t n_jobs, const int *n_seq, const int *seq_lens,
                          const uint8_t *seqs, const int *progressive, uint8_t **msa_out, int *msa_len,
                          int64_t *cells);

/* Trace form of barb200_poa_msa_batch: the same jobs, dealt over the context's devices the same way, through trace kernels that also
 * record every alignment the device makes. trace_out[i] = malloc'd array of n_words[i] int64 words (release with barb200_free):
 *   n_seq, msa_len, cells                          (cells as barb200_poa_msa_batch returns them)
 *   read_id_map[n_seq]                             the read order (guide tree): read_id_map[a] = the job's read aligned a-th
 *   per alignment a (n_seq records, in read order):
 *     read_id, qlen, node_n (before the alignment), n_cigar, best_score, n_rows (= node_n - 1; 0 for the first read, which
 *     starts the graph and is not aligned; its n_cigar and best_score are 0 too)
 *     cigar[n_cigar]                               abPOA's graph cigar words (uint64 stored as int64)
 *     dp_beg[n_rows], dp_end[n_rows]               the adaptive band of every DP row, in topological order
 *   the MSA, n_seq x msa_len bytes row-major, packed 8 bytes per word (the last word padded with zeros)
 * This is the layout abPOA's own per-alignment state gives (abpoa_align_sequence_to_subgraph's graph_cigar and best score,
 * abm->dp_beg / dp_end), so that a device run can be compared with the reference alignment by alignment. The MSAs and cells are
 * those of barb200_poa_msa_batch. Errors as barb200_poa_msa_batch: on failure no arrays are left. For tests and diagnosis; its speed
 * is not a goal. */
int barb200_poa_trace_batch(barb200_ctx *ctx, int64_t n_jobs, const int *n_seq, const int *seq_lens, const uint8_t *seqs,
                            const int *progressive, int64_t **trace_out, int64_t *n_words);

/* Trace form of barb200_make_consistent_partial_order_alignments (arguments as barb200_flower_submit; right_end_indexes == NULL:
 * independent ends): every sliding window of every end, window by window. Window n+1 of an end is cut at offsets that window n's
 * trimmed MSA decides, so a window cannot be checked on its own; this call records the whole chain. trace_out[e] = malloc'd array
 * of n_words[e] int64 words per end (release each with barb200_free), K = the end's string count:
 *   K, n_windows                                   (no windows for a single string or an end without bases)
 *   per window, in chain order:
 *     window index (0, 1, ...)
 *     offset[K]                                    where each row's slice starts in its string
 *     len[K]                                       the slice lengths the POA job gets (1 for a row given the N stand-in)
 *     empty[K]                                     1: the row ran out of bases and got the N stand-in (poaBarAligner.c:551-562)
 *     progressive                                  the job's progressive flag (:567-571)
 *     n_trace, trace[n_trace]                      the window's POA job, word for word in barb200_poa_trace_batch's layout
 *     trimmed_len[K], column_no                    the window's row lengths and columns after trimming against both neighbours,
 *                                                  as the stitch uses them
 *   K, column_no, the end's MSA                    stitched and trimmed across ends: barb200_make_consistent_partial_order_
 *                                                  alignments' MSA, K x column_no bytes row-major, packed 8 bytes per word
 * The windows run through the same window, trim and stitch steps as the end queue, in synchronous rounds (the next window of every
 * unfinished end in one trace call), not through the queue's batches: a window's result depends on its job alone. Not covered:
 * the production kernels' node order (traces number rows in abPOA's BFS order, as barb200_poa_trace_batch does) and the queue's
 * batching, which the final MSAs check. Errors as barb200_make_consistent_partial_order_alignments, with its messages; the return
 * is a BARB200_* code and on failure no arrays are left. For diagnosis; its speed is not a goal. */
int barb200_trace_ends(barb200_ctx *ctx, int64_t end_no, const int64_t *end_lengths, char ***end_strings,
                       int **end_string_lengths, int64_t **right_end_indexes, int64_t **right_end_row_indexes, int64_t **overlaps,
                       int64_t window_size, int64_t max_prog_rows, double max_prog_length_diff, int64_t **trace_out,
                       int64_t *n_words);

/* Staged form of the same call for callers (and bench.py) that keep inputs resident in HBM:
 * stage = host packing + guide trees + H2D once; run = kernel(s) only, may be repeated; fetch = D2H + unpack. */
typedef struct barb200_stage barb200_stage;
int barb200_stage_create(barb200_ctx *ctx, int64_t n_jobs, const int *n_seq, const int *seq_lens,
                         const uint8_t *seqs, const int *progressive, barb200_stage **out);
int barb200_stage_run(barb200_stage *st, float *kernel_ms /* may be NULL: device time of the launch(es) */);
int barb200_stage_fetch(barb200_stage *st, uint8_t **msa_out, int *msa_len, int64_t *cells);
int64_t barb200_stage_launches(barb200_stage *st);   /* kernels launched by the last barb200_stage_run */
/* per-phase SM clock totals of the last run over all POA CTAs (needs collect_phase_clocks): dp, backtrack, fuse, topo, msa, total;
 * out[6] = device time of the guide-tree kernel (K0) in nanoseconds (always filled) */
int barb200_stage_phase_clocks(barb200_stage *st, uint64_t out[7]);
/* the stage's CTA-size buckets (largest first): out[4b .. 4b+3] = threads per CTA, jobs, resident CTAs, plane ints per slot;
 * returns the number of buckets */
int barb200_stage_buckets(barb200_stage *st, int64_t *out, int max_buckets);
void barb200_stage_destroy(barb200_stage *st);

/* The reference's Msa (bar/inc/poaBarAligner.h:37-43) with one flat matrix instead of row pointers. */
typedef struct {
    int64_t seq_no;
    int64_t column_no;
    int *seq_lens;       /* [seq_no] input lengths (as the reference's Msa.seq_lens after stitching) */
    uint8_t *msa;        /* [seq_no * column_no] 0-3 ACGT, 4 N, 5 gap */
} barb200_msa;
void barb200_msa_destruct(barb200_msa *m);

/* msa_make_partial_order_alignment for n_ends independent ends at once. seqs[e][i] is the i-th ASCII string of end e
 * (not necessarily NUL terminated), seq_lens[e][i] its length, seq_no[e] the number of strings.
 * out[e] receives a new barb200_msa. Inputs are not retained. */
int barb200_msa_make_partial_order_alignment_batch(barb200_ctx *ctx, int64_t n_ends, const int64_t *seq_no,
        char ***seqs, int **seq_lens, int64_t window_size, int64_t max_prog_rows, double max_prog_length_diff,
        barb200_msa **out);

/* Single-end convenience with the reference's argument order (bar/inc/poaBarAligner.h:76). */
barb200_msa *barb200_msa_make_partial_order_alignment(barb200_ctx *ctx, char **seqs, int *seq_lens, int64_t seq_no,
        int64_t window_size, int64_t max_prog_rows, double max_prog_length_diff);

/* make_consistent_partial_order_alignments (bar/inc/poaBarAligner.h:108): same arguments, abpoa_para_t replaced by
 * the context. Returns a malloc'd array of end_no barb200_msa* (release each with barb200_msa_destruct and the array
 * with barb200_free), or NULL on error. */
barb200_msa **barb200_make_consistent_partial_order_alignments(barb200_ctx *ctx, int64_t end_no, int64_t *end_lengths,
        char ***end_strings, int **end_string_lengths, int64_t **right_end_indexes, int64_t **right_end_row_indexes,
        int64_t **overlaps, int64_t window_size, int64_t max_prog_rows, double max_prog_length_diff);

/* ------------------------------------------------------------------------------------------------------------
 * cPecan mode (bar/partialOrderAlignment="0"): the banded five-state pair-HMM posteriors.
 *
 *   - barb200_pecan_aligned_pairs_batch replaces getAlignedPairsUsingAnchors
 *     (submodules/cPecan/inc/pairwiseAligner.h, impl/pairwiseAligner.c:1477-1495), the call
 *     addMultipleAlignedPairs makes once per chosen sequence pair (impl/multipleAligner.c:660, via getAlignedPairs
 *     :1527-1534), for MANY sequence pairs at once: split at large anchor gaps (getSplitPoints :1265-1292), banded
 *     forward / backward / posterior match probabilities (getPosteriorProbsWithBanding :766-887), coordinates shifted
 *     back (:1457-1464). Anchors stay the caller's (getAnchorPairsForPairwiseAlignmentParameters :1222-1233).
 *   - barb200_pecan_params are the PairwiseAlignmentParameters fields that path reads
 *     (pairwiseAlignmentBandingParameters_construct :1369-1391; bar/impl/bar.c:20-37 for the <bar><pecan> keys).
 *   The state machine is the reference's fiveState machine with its built-in constants (stateMachine.c:482-521).
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
    double threshold;                      /* 0.01 */
    int64_t min_diags_between_traceback;   /* 1000 */
    int64_t traceback_diagonals;           /* 40 */
    int64_t diagonal_expansion;            /* 20; <bar><pecan diagonalExpansion> */
    int64_t split_matrix_bigger_than_this; /* 3000*3000; <bar><pecan splitMatrixBiggerThanThis> SQUARED as bar.c:23-24 does */
    int dynamic_anchor_expansion;          /* must be 0 (band_constructDynamic is not used by Cactus) */
} barb200_pecan_params;
void barb200_pecan_params_default(barb200_pecan_params *p);

/* For pair i: NUL-free ASCII strings sx[i] (length lx[i]) and sy[i] (ly[i]); anchors[i] = n_anchor[i] (x, y) pairs of
 * 0-based sequence coordinates, strictly increasing in both (may be NULL when n_anchor[i] == 0); ragged_left[i] /
 * ragged_right[i] as alignmentHasRaggedLeftEnd / RightEnd. Outputs per pair: triples_out[i] = malloc'd n_out[i] x 3
 * int64 (score = floor(posterior * PAIR_ALIGNMENT_PROB_1), x, y) in the order the reference returns them;
 * posteriors_out (may be NULL) receives malloc'd doubles, the pre-floor posteriors exp(f_M + b_M - total);
 * cells_out (may be NULL) the banded DP cells of the pair (sum of diagonal widths over its sub-matrices).
 * Release every array with barb200_free.
 * Several devices (barb200_params.n_devices): whole pairs are dealt to the context's devices by their banded cells and every
 * device runs its share at once; the outputs are those of a single-device context, bit for bit. If any device fails, the call
 * fails with that device's message and leaves no outputs. */
int barb200_pecan_aligned_pairs_batch(barb200_ctx *ctx, const barb200_pecan_params *p, int64_t n_pairs,
                                      const char *const *sx, const int64_t *lx, const char *const *sy, const int64_t *ly,
                                      const int64_t *const *anchors, const int64_t *n_anchor,
                                      const uint8_t *ragged_left, const uint8_t *ragged_right,
                                      int64_t **triples_out, int64_t *n_out, double **posteriors_out, int64_t *cells_out);

/* Staged form (inputs resident in HBM; used by bench.py): create = split + band + pack + H2D; run = kernels only
 * (repeatable); fetch = compaction + D2H + exp/threshold/floor on the host. A stage lives on the context's first device,
 * whatever the number of devices. */
typedef struct barb200_pecan_stage barb200_pecan_stage;
int barb200_pecan_stage_create(barb200_ctx *ctx, const barb200_pecan_params *p, int64_t n_pairs,
                               const char *const *sx, const int64_t *lx, const char *const *sy, const int64_t *ly,
                               const int64_t *const *anchors, const int64_t *n_anchor,
                               const uint8_t *ragged_left, const uint8_t *ragged_right, barb200_pecan_stage **out);
int barb200_pecan_stage_run(barb200_pecan_stage *st, float *kernel_ms);
int barb200_pecan_stage_fetch(barb200_pecan_stage *st, int64_t **triples_out, int64_t *n_out, double **posteriors_out,
                              int64_t *cells_out);
int64_t barb200_pecan_stage_cells(barb200_pecan_stage *st);      /* banded cells of the whole stage */
int64_t barb200_pecan_stage_launches(barb200_pecan_stage *st);   /* kernels launched by the last run */
void barb200_pecan_stage_destroy(barb200_pecan_stage *st);

/* Host-only planning helper (no device work): the band of one sub-matrix as the engine builds it -- xmyL / xmyR of the
 * diagonals 0..lx+ly (band_construct, pairwiseAligner.c:193-244). Returns 0 or BARB200_EINVAL. */
int barb200_pecan_band(int64_t lx, int64_t ly, const int64_t *anchors, int64_t n_anchor, int64_t expansion,
                       int64_t *xmy_l, int64_t *xmy_r);
/* Host-only: getSplitPoints (pairwiseAligner.c:1265-1292). splits_out = malloc'd n x 4 (x1, y1, x2, y2); returns n or <0. */
int64_t barb200_pecan_split_points(int64_t lx, int64_t ly, const int64_t *anchors, int64_t n_anchor,
                                   int64_t split_matrix_bigger_than_this, int ragged_left, int ragged_right,
                                   int64_t **splits_out);

/* ------------------------------------------------------------------------------------------------------------
 * cPecan mode's anchors: the MUM chains of getAnchorPairsForPairwiseAlignmentParameters with useMumAnchors = 1
 * (submodules/cPecan/impl/pairwiseAligner.c:1222-1231 -> getAlignedMums :1849-2121), which addMultipleAlignedPairs computes
 * for every sequence pair before its posteriors (getAlignedPairs :1527-1534).
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
    int64_t k;                              /* 50; k-mer length, 1..64 */
    int64_t u;                              /* 1; a match must be longer than u + either neighbour's in Y's k-mer order */
    int64_t anchor_matrix_bigger_than_this; /* 500*500; <bar><pecan anchorMatrixBiggerThanThis> SQUARED as bar.c:25-26 does */
    int recursive_mums;                     /* 1; one non-recursive level into every gap of the chain larger than the above */
} barb200_mum_params;
void barb200_mum_params_default(barb200_mum_params *p);

/* For pair i: NUL-free 7-bit ASCII strings sx[i] (length lx[i]) and sy[i] (ly[i]). anchors_out[i] = malloc'd n_anchor_out[i] x 2
 * int64 (x, y), 0-based, in the reference's order -- strictly increasing in both with recursive_mums (what
 * barb200_pecan_aligned_pairs_batch takes), last MUM first and each MUM backwards without. Release with barb200_free.
 * BARB200_EINVAL for k outside 1..64, u < 0, or a NUL / non-ASCII byte.
 * Several devices: the pairs larger than anchor_matrix_bigger_than_this are dealt to the context's devices by the device memory
 * they take, and every device runs its share at once; the anchors are those of a single-device context. */
int barb200_pecan_anchor_pairs_batch(barb200_ctx *ctx, const barb200_mum_params *p, int64_t n_pairs,
                                     const char *const *sx, const int64_t *lx, const char *const *sy, const int64_t *ly,
                                     int64_t **anchors_out, int64_t *n_anchor_out);
/* The calling thread's last barb200_pecan_anchor_pairs_batch: out[0] device time of its kernels and copies (ms; with several
 * devices, that of the device that took longest), out[1] wall time of the call (ms), out[2] kernels launched on all devices.
 * For reports. */
int barb200_mum_last_timing(double out[3]);

/* Per device of the context (up to max_devices entries; either array may be NULL): the sequence pairs
 * barb200_pecan_aligned_pairs_batch (hmm_pairs) and barb200_pecan_anchor_pairs_batch (mum_pairs, only pairs that needed the
 * device) have run there since the context was created; the staged form is not counted. Returns the number of devices of the
 * context. For reports and tests. */
int barb200_pecan_device_stats(barb200_ctx *ctx, int64_t *hmm_pairs, int64_t *mum_pairs, int max_devices);

/* ------------------------------------------------------------------------------------------------------------
 * The end queue, asynchronously. barb200_flower_submit takes the arguments of make_consistent_partial_order_alignments
 * (bar/inc/poaBarAligner.h:108; right_end_indexes == NULL: independent ends, no cross-end trimming -- the single-end case of
 * make_flower_alignment_poa, poaBarAligner.c:1119-1143), copies what it needs and returns at once; the strings may be released
 * after the call. barb200_flower_wait blocks until every end of the ticket is aligned, does the stitching and the cross-end
 * trimming in the calling thread and returns what barb200_make_consistent_partial_order_alignments returns (NULL + last_error on
 * failure; a failure of one ticket does not affect the others). The ticket is consumed by the wait.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct barb200_ticket barb200_ticket;
barb200_ticket *barb200_flower_submit(barb200_ctx *ctx, int64_t end_no, const int64_t *end_lengths, char ***end_strings,
        int **end_string_lengths, int64_t **right_end_indexes, int64_t **right_end_row_indexes, int64_t **overlaps,
        int64_t window_size, int64_t max_prog_rows, double max_prog_length_diff);
barb200_msa **barb200_flower_wait(barb200_ctx *ctx, barb200_ticket *ticket);
/* device batches the queue has run so far and the jobs in them (reports, tests) */
int barb200_queue_stats(barb200_ctx *ctx, int64_t *batches, int64_t *jobs);

/* Host-side phases of the context's most recent device batch, in milliseconds: out[0] build (pack, validation, planning, H2D),
 * out[1] launch + wait, out[2] device time of the kernels, out[3] fetch (D2H + unpack), out[4] total,
 * out[5] = number of jobs. For reports (bench.py's per-phase breakdown). */
int barb200_last_batch_timing(barb200_ctx *ctx, double out[6]);

/* Device facts for reports. */
int barb200_device_count(barb200_ctx *ctx);
int barb200_device_info(barb200_ctx *ctx, int *sm_count, int64_t *mem_total, int64_t *mem_free, char *name, int name_len);

void barb200_free(void *p);
/* barb200_free on n pointers (the MSAs of a batch), and a parallel gather of n buffers into one (rows[i], bytes[i]) -> dst: what a
 * caller in a scripting language would otherwise do one foreign call at a time. */
void barb200_free_many(void *const *p, int64_t n);
void barb200_pack_rows(void *const *rows, const int64_t *bytes, int64_t n, uint8_t *dst);

#ifdef __cplusplus
}
#endif
#endif
