/*
 * cactus_bar_shim.c -- the thin C host shim between Cactus' BAR code and libbarb200 (include/barb200.h).
 *
 * Compiled AGAINST THE CACTUS TREE (bar/inc/poaBarAligner.h and what it includes) and linked into cactusBarLib.a in
 * place of the two reference functions it re-exports with their reference signatures:
 *
 *     Msa  *msa_make_partial_order_alignment(...)            bar/inc/poaBarAligner.h:76,  bar/impl/poaBarAligner.c:463-749
 *     Msa **make_consistent_partial_order_alignments(...)    bar/inc/poaBarAligner.h:108, bar/impl/poaBarAligner.c:751-801
 *
 * Everything above them -- bar() (bar/impl/bar.c:52), make_flower_alignment_poa (poaBarAligner.c:1115), the
 * Flower/End/Cap/CactusDisk API, CAF -- stays the reference's code and keeps calling these two symbols, so
 * cactus_consolidated and the Python/Toil pipeline run unchanged. See INTEGRATION.md for the build hook.
 *
 * Semantics kept: ownership (the returned Msa owns seqs / seq_lens exactly as the reference's does,
 * poaBarAligner.c:474-475, 708-717; released by the reference's msa_destruct), re-entrancy (called concurrently from
 * OpenMP teams, bar.c:90-94, poaBarAligner.c:772 -- calls are funnelled into one engine context, which serialises
 * device batches), error convention (no return codes: failure -> st_errAbort, i.e. message + exit(1), as every
 * other fatal condition in this code path).
 * There is no CPU fallback: if no CUDA device is usable the process aborts with the engine's message.
 */
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include "poaBarAligner.h"
#include "barb200.h"
#include "barb200_shim_env.h"

static pthread_mutex_t shim_mutex = PTHREAD_MUTEX_INITIALIZER;
/* one engine per distinct parameter set, created on first use and kept for the life of the process: another OpenMP thread
 * may be inside a call on any of them, so a context is never destroyed or replaced in place */
#define SHIM_MAX_CTX 16
static struct { barb200_params p; barb200_ctx *ctx; } shim_ctxs[SHIM_MAX_CTX];
static int shim_ctx_no = 0;

/* abpoa_para_t (as built by abpoaParamaters_constructFromCactusParams, poaBarAligner.c:24-81) -> barb200_params */
static void params_from_abpoa(const abpoa_para_t *abpt, barb200_params *p) {
    barb200_params_default(p);
    memcpy(p->mat, abpt->mat, 25 * sizeof(int));
    p->gap_open1 = abpt->gap_open1; p->gap_ext1 = abpt->gap_ext1;
    p->gap_open2 = abpt->gap_open2; p->gap_ext2 = abpt->gap_ext2;
    p->wb = abpt->wb; p->wf = abpt->wf;
    p->k = abpt->k; p->w = abpt->w; p->min_w = abpt->min_w;
    p->progressive_poa = abpt->progressive_poa;
    p->disable_seeding = abpt->disable_seeding;
    barb200_devices_from_env(p);                          /* BARB200_DEVICE / BARB200_DEVICES */
}

/* field-wise comparison (memcmp would read struct padding) */
static int params_equal(const barb200_params *a, const barb200_params *b) {
    return memcmp(a->mat, b->mat, sizeof(a->mat)) == 0 && a->gap_open1 == b->gap_open1 && a->gap_ext1 == b->gap_ext1 &&
           a->gap_open2 == b->gap_open2 && a->gap_ext2 == b->gap_ext2 && a->wb == b->wb && a->wf == b->wf && a->k == b->k &&
           a->w == b->w && a->min_w == b->min_w && a->progressive_poa == b->progressive_poa &&
           a->disable_seeding == b->disable_seeding && a->device == b->device && a->n_devices == b->n_devices &&
           memcmp(a->devices, b->devices, sizeof(a->devices)) == 0;
}

static barb200_ctx *shim_context(abpoa_para_t *abpt) {
    barb200_params p;
    params_from_abpoa(abpt, &p);
    pthread_mutex_lock(&shim_mutex);
    for (int i = 0; i < shim_ctx_no; i++) {
        if (params_equal(&p, &shim_ctxs[i].p)) {
            barb200_ctx *ctx = shim_ctxs[i].ctx;
            pthread_mutex_unlock(&shim_mutex);
            return ctx;
        }
    }
    if (shim_ctx_no == SHIM_MAX_CTX) {
        pthread_mutex_unlock(&shim_mutex);
        st_errAbort("barb200: more than %d distinct POA parameter sets in one process", SHIM_MAX_CTX);
    }
    char err[256];
    barb200_ctx *ctx = barb200_create(&p, err, (int)sizeof(err));
    if (ctx == NULL) {
        pthread_mutex_unlock(&shim_mutex);
        st_errAbort("barb200: cannot create the GPU BAR engine: %s", err);
    }
    shim_ctxs[shim_ctx_no].p = p;
    shim_ctxs[shim_ctx_no].ctx = ctx;
    shim_ctx_no++;
    pthread_mutex_unlock(&shim_mutex);
    return ctx;
}

/* barb200_msa (flat matrix) -> the reference's Msa (row pointers); takes ownership of the caller's
 * seqs / seq_lens like the reference (seq_lens keeps the input lengths, poaBarAligner.c:708-717) */
static Msa *msa_from_engine(barb200_msa *m, char **seqs, int *seq_lens) {
    Msa *msa = st_malloc(sizeof(Msa));
    msa->seq_no = m->seq_no;
    msa->seqs = seqs;
    msa->seq_lens = seq_lens;
    msa->column_no = (int)m->column_no;
    msa->msa_seq = st_malloc(sizeof(uint8_t *) * (m->seq_no > 0 ? m->seq_no : 1));
    for (int64_t i = 0; i < m->seq_no; i++) {
        msa->msa_seq[i] = st_malloc(m->column_no > 0 ? m->column_no : 1);
        memcpy(msa->msa_seq[i], m->msa + i * m->column_no, m->column_no);
    }
    barb200_msa_destruct(m);
    return msa;
}

Msa *msa_make_partial_order_alignment(char **seqs, int *seq_lens, int64_t seq_no, int64_t window_size,
                                      int64_t max_prog_rows, double max_prog_length_diff, abpoa_para_t *poa_parameters) {
    barb200_ctx *ctx = shim_context(poa_parameters);
    barb200_msa *m = barb200_msa_make_partial_order_alignment(ctx, seqs, seq_lens, seq_no, window_size, max_prog_rows,
                                                              max_prog_length_diff);
    if (m == NULL) {
        st_errAbort("barb200: msa_make_partial_order_alignment failed: %s", barb200_last_error(ctx));
    }
    return msa_from_engine(m, seqs, seq_lens);
}

Msa **make_consistent_partial_order_alignments(int64_t end_no, int64_t *end_lengths, char ***end_strings,
        int **end_string_lengths, int64_t **right_end_indexes, int64_t **right_end_row_indexes, int64_t **overlaps,
        int64_t window_size, int64_t max_prog_rows, double max_prog_length_diff, abpoa_para_t *poa_parameters) {
    barb200_ctx *ctx = shim_context(poa_parameters);
    /* all ends of the flower in ONE batched device call (the reference loops, optionally with a nested OpenMP team) */
    barb200_msa **ms = barb200_make_consistent_partial_order_alignments(ctx, end_no, end_lengths, end_strings,
            end_string_lengths, right_end_indexes, right_end_row_indexes, overlaps, window_size, max_prog_rows,
            max_prog_length_diff);
    if (ms == NULL) {
        st_errAbort("barb200: make_consistent_partial_order_alignments failed: %s", barb200_last_error(ctx));
    }
    Msa **msas = st_malloc(sizeof(Msa *) * (end_no > 0 ? end_no : 1));
    for (int64_t i = 0; i < end_no; i++) {
        msas[i] = msa_from_engine(ms[i], end_strings[i], end_string_lengths[i]);
    }
    barb200_free(ms);
    return msas;
}

#ifdef CACTUS_BAR_B200_BAR
/* ---------------------------------------------------------------------------------------------------------------------
 * bar() with a global end queue (SURVEY.md 8(f)-2). The reference's bar() (bar/impl/bar.c:52-176) aligns one flower per OpenMP
 * thread and only then runs CAF on it, so the device never sees more than `threads` flowers at once. Here the loop is split:
 *   pass 1  every leaf flower's end strings are extracted (the reference's own get_end_sequences / getDominantEnd, exactly as
 *           make_flower_alignment_poa does, poaBarAligner.c:1115-1196) and SUBMITTED to the engine's end queue;
 *   pass 2  per flower: wait for its alignments, create_alignment_blocks, then the CAF steps of bar.c:119-164 unchanged --
 *           on the CPU threads, while the GPU works through the ends of the flowers further down the list.
 * Built with -DCACTUS_BAR_B200_BAR; the reference's own bar() is kept as bar_reference (objcopy --redefine-sym bar=bar_reference
 * on bar.o, or a #define in bar.c) and serves the cPecan configuration (partialOrderAlignment="0").
 * --------------------------------------------------------------------------------------------------------------------- */
#include "cactus.h"
#include "flowerAligner.h"
#include "stCaf.h"
#include "stPinchGraphs.h"
#include "stPinchIterator.h"
#if defined(_OPENMP)
#include <omp.h>
#endif

void bar_reference(stList *flowers, CactusParams *params, CactusDisk *cactusDisk, stList *listOfEndAlignmentFiles);
/* defined (not static) in the reference's poaBarAligner.c / bar.c but not declared in their headers */
void get_end_sequences(End *end, char **end_strings, int *end_string_lengths, int64_t *overlaps, Cap **indices_to_caps,
                       int64_t max_seq_length, int64_t mask_filter);
int64_t getMaxSequenceLength(End *end);
void create_alignment_blocks(Msa *msa, Cap **row_indexes_to_caps, stList *alignment_blocks);
bool blockFilterFn(stPinchBlock *pinchBlock, void *extraArg);

typedef struct {
    int64_t end_no;                     /* 1 in the dominant-end case */
    bool dominant;
    int64_t *end_lengths;
    char ***end_strings;
    int **end_string_lengths;
    int64_t **right_end_indexes, **right_end_row_indexes, **overlaps;
    Cap ***indices_to_caps;
    barb200_ticket *ticket;
} FlowerPlan;

/* the first half of make_flower_alignment_poa (poaBarAligner.c:1115-1196): strings and indexes of every end, then submit */
static void plan_flower(FlowerPlan *fp, barb200_ctx *ctx, Flower *flower, int64_t max_seq_length, int64_t window_size, int64_t mask_filter,
                        int64_t max_prog_rows, double max_prog_length_diff) {
    End *dominantEnd = getDominantEnd(flower);
    fp->dominant = dominantEnd != NULL && getMaxSequenceLength(dominantEnd) < max_seq_length;
    fp->end_no = fp->dominant ? 1 : flower_getEndNumber(flower);
    int64_t n = fp->end_no > 0 ? fp->end_no : 1;
    fp->end_lengths = st_calloc(n, sizeof(int64_t));
    fp->end_strings = st_calloc(n, sizeof(char **));
    fp->end_string_lengths = st_calloc(n, sizeof(int *));
    fp->right_end_indexes = st_calloc(n, sizeof(int64_t *));
    fp->right_end_row_indexes = st_calloc(n, sizeof(int64_t *));
    fp->overlaps = st_calloc(n, sizeof(int64_t *));
    fp->indices_to_caps = st_calloc(n, sizeof(Cap **));
    if (fp->dominant) {                                             /* :1119-1143 */
        int64_t seq_no = end_getInstanceNumber(dominantEnd);
        fp->end_lengths[0] = seq_no;
        fp->end_strings[0] = st_malloc(sizeof(char *) * seq_no);
        fp->end_string_lengths[0] = st_malloc(sizeof(int) * seq_no);
        fp->overlaps[0] = st_malloc(sizeof(int64_t) * seq_no);
        fp->indices_to_caps[0] = st_malloc(sizeof(Cap *) * seq_no);
        get_end_sequences(dominantEnd, fp->end_strings[0], fp->end_string_lengths[0], fp->overlaps[0], fp->indices_to_caps[0],
                          max_seq_length, mask_filter);
    } else {                                                        /* :1145-1196 */
        stHash *caps_to_indices = stHash_construct2(NULL, free);
        End *end;
        Flower_EndIterator *endIterator = flower_getEndIterator(flower);
        int64_t i = 0;
        while ((end = flower_getNextEnd(endIterator)) != NULL) {
            int64_t k = end_getInstanceNumber(end);
            fp->end_lengths[i] = k;
            fp->end_strings[i] = st_malloc(sizeof(char *) * k);
            fp->end_string_lengths[i] = st_malloc(sizeof(int) * k);
            fp->right_end_indexes[i] = st_malloc(sizeof(int64_t) * k);
            fp->right_end_row_indexes[i] = st_malloc(sizeof(int64_t) * k);
            fp->indices_to_caps[i] = st_malloc(sizeof(Cap *) * k);
            fp->overlaps[i] = st_malloc(sizeof(int64_t) * k);
            get_end_sequences(end, fp->end_strings[i], fp->end_string_lengths[i], fp->overlaps[i], fp->indices_to_caps[i],
                              max_seq_length, mask_filter);
            for (int64_t j = 0; j < k; j++) {
                stHash_insert(caps_to_indices, fp->indices_to_caps[i][j], stIntTuple_construct2(i, j));
            }
            i++;
        }
        flower_destructEndIterator(endIterator);
        for (i = 0; i < fp->end_no; i++) {
            for (int64_t j = 0; j < fp->end_lengths[i]; j++) {
                Cap *cap2 = cap_getReverse(cap_getAdjacency(fp->indices_to_caps[i][j]));
                stIntTuple *k = stHash_search(caps_to_indices, cap2);
                assert(k != NULL);
                fp->right_end_indexes[i][j] = stIntTuple_get(k, 0);
                fp->right_end_row_indexes[i][j] = stIntTuple_get(k, 1);
            }
        }
        stHash_destruct(caps_to_indices);
    }
    fp->ticket = barb200_flower_submit(ctx, fp->end_no, fp->end_lengths, fp->end_strings, fp->end_string_lengths,
                                       fp->dominant ? NULL : fp->right_end_indexes, fp->dominant ? NULL : fp->right_end_row_indexes,
                                       fp->dominant ? NULL : fp->overlaps, window_size, max_prog_rows, max_prog_length_diff);
    if (fp->ticket == NULL) {
        st_errAbort("barb200: submitting a flower's ends failed: %s", barb200_last_error(ctx));
    }
}

/* the second half (:1198-1236): alignments -> alignment blocks, in the reference's order */
static stList *finish_flower(FlowerPlan *fp, barb200_ctx *ctx) {
    barb200_msa **ms = barb200_flower_wait(ctx, fp->ticket);
    if (ms == NULL) {
        st_errAbort("barb200: aligning a flower's ends failed: %s", barb200_last_error(ctx));
    }
    stList *alignment_blocks = stList_construct3(0, (void (*)(void *)) alignmentBlock_destruct);
    for (int64_t i = 0; i < fp->end_no; i++) {
        Msa *msa = msa_from_engine(ms[i], fp->end_strings[i], fp->end_string_lengths[i]);    /* owns the strings from here on */
        create_alignment_blocks(msa, fp->indices_to_caps[i], alignment_blocks);
        msa_destruct(msa);
        free(fp->right_end_indexes[i]);
        free(fp->right_end_row_indexes[i]);
        free(fp->indices_to_caps[i]);
        free(fp->overlaps[i]);
    }
    barb200_free(ms);
    free(fp->end_lengths); free(fp->end_strings); free(fp->end_string_lengths);
    free(fp->right_end_indexes); free(fp->right_end_row_indexes); free(fp->overlaps); free(fp->indices_to_caps);
    return alignment_blocks;
}

void bar(stList *flowers, CactusParams *params, CactusDisk *cactusDisk, stList *listOfEndAlignmentFiles) {
    if (!cactusParams_get_int(params, 2, "bar", "partialOrderAlignment")) {
        bar_reference(flowers, params, cactusDisk, listOfEndAlignmentFiles);       /* cPecan configuration */
        return;
    }
    /* the parameters bar() reads for the POA configuration, bar.c:57-74 */
    int64_t maximumLength = cactusParams_get_int(params, 2, "bar", "bandingLimit");
    int64_t poaWindow = cactusParams_get_int(params, 3, "bar", "poa", "partialOrderAlignmentWindow");
    int64_t maskFilter = cactusParams_get_int(params, 3, "bar", "poa", "partialOrderAlignmentMaskFilter");
    int64_t poaMaxProgRows = cactusParams_get_int(params, 3, "bar", "poa", "partialOrderAlignmentProgressiveMaxRows");
    double poaMaxLenDiff = cactusParams_get_float(params, 3, "bar", "poa", "partialOrderAlignmentProgressiveMaxLengthDiff");
    abpoa_para_t *poaParameters = abpoaParamaters_constructFromCactusParams(params);
    if (listOfEndAlignmentFiles != NULL && stList_length(flowers) != 1) {
        st_errAbort("We have precomputed alignments but %" PRIi64 " flowers to align.\n", stList_length(flowers));
    }
    barb200_ctx *ctx = shim_context(poaParameters);
    int64_t flowerNo = stList_length(flowers);
    FlowerPlan *plans = st_calloc(flowerNo > 0 ? flowerNo : 1, sizeof(FlowerPlan));

    /* pass 1: every end of every leaf flower goes into the queue */
#if defined(_OPENMP)
#pragma omp parallel for schedule(dynamic, 1)
#endif
    for (int64_t j = 0; j < flowerNo; j++) {
        plan_flower(&plans[j], ctx, stList_get(flowers, j), maximumLength, poaWindow, maskFilter, poaMaxProgRows, poaMaxLenDiff);
    }

    /* pass 2: collect flower by flower; CAF (bar.c:96-164, unchanged) overlaps the device work of the flowers still queued */
#if defined(_OPENMP)
#pragma omp parallel for schedule(dynamic, 1)
#endif
    for (int64_t j = 0; j < flowerNo; j++) {
        Flower *flower = stList_get(flowers, j);
        FilterArgs *fa = st_calloc(1, sizeof(FilterArgs));
        fa->minimumIngroupDegree = cactusParams_get_int(params, 2, "bar", "minimumIngroupDegree");
        fa->minimumOutgroupDegree = cactusParams_get_int(params, 2, "bar", "minimumOutgroupDegree");
        fa->minimumDegree = cactusParams_get_int(params, 2, "bar", "minimumBlockDegree");
        fa->minimumNumberOfSpecies = cactusParams_get_int(params, 2, "bar", "minimumNumberOfSpecies");
        fa->flower = flower;

        stList *alignments = finish_flower(&plans[j], ctx);
        st_logDebug("Created the poa alignments: %" PRIi64 " poa alignment blocks for flower\n", stList_length(alignments));
        stPinchIterator *pinchIterator = stPinchIterator_constructFromAlignedBlocks(alignments);

        stPinchThreadSet *threadSet = stCaf_setup(flower);
        stCaf_anneal(threadSet, pinchIterator, NULL, flower);
        if (fa->minimumDegree < 2) {
            stCaf_makeDegreeOneBlocks(threadSet);
        }
        if (fa->minimumIngroupDegree > 0 || fa->minimumOutgroupDegree > 0 || fa->minimumDegree > 1) {
            stCaf_melt(flower, threadSet, blockFilterFn, fa, 0, 0, 0, INT64_MAX);
        }
        stCaf_finish(flower, threadSet, INT64_MAX, INT64_MAX);
        stPinchThreadSet_destruct(threadSet);
        stPinchIterator_destruct(pinchIterator);
        stList_destruct(alignments);
        free(fa);
    }
    free(plans);
    abpoa_free_para(poaParameters);
}
#endif /* CACTUS_BAR_B200_BAR */
