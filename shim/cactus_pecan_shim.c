/*
 * cactus_pecan_shim.c -- the thin C host shim between cPecan's multiple aligner (used by Cactus' BAR phase when
 * bar/partialOrderAlignment="0") and libbarb200's pair-HMM engine (include/barb200.h, barb200_pecan_*).
 *
 * Compiled AGAINST THE CACTUS TREE (submodules/cPecan/inc + sonLib) and linked into cPecanLib.a in place of the two
 * reference functions it re-exports with their reference signatures:
 *
 *   stList *getAlignedPairsUsingAnchors(StateMachine*, const char *sX, const char *sY, stList *anchorPairs,
 *                                       PairwiseAlignmentParameters*, bool raggedLeft, bool raggedRight)
 *        submodules/cPecan/inc/pairwiseAligner.h, impl/pairwiseAligner.c:1477-1495 -- one pair per call (a batch of one:
 *        correct, but a single warp of the GPU works);
 *   stList *makeAllPairwiseAlignments(StateMachine*, stList *seqFrags, PairwiseAlignmentParameters*, stList **scores)
 *        inc/multipleAligner.h:75, impl/multipleAligner.c:667-680 -- ALL sequence pairs of an end in one device batch
 *        (this is the call makeAlignmentUsingAllPairs issues, multipleAligner.c:690, i.e. what makeAlignment does
 *        whenever spanningTrees * (n-1) >= n(n-1)/2, :893-895).
 *
 * Anchors of a round of pairs: with useMumAnchors (Cactus' default) one barb200_pecan_anchor_pairs_batch call, the device's
 * restatement of getAnchorPairsForPairwiseAlignmentParameters (pairwiseAligner.c:1222-1231: MUM chains); otherwise (the lastz
 * path) the reference's own code on the host. Everything above stays the reference's: makeAlignment's pair selection, the poset alignment, endAligner.c,
 * flowerAligner.c, bar(). The state machine must be the reference's five-state machine with its built-in constants
 * (stateMachine5_construct(fiveState), the one bar() builds at bar/impl/bar.c:66); anything else aborts.
 *
 * Error convention as the reference's: st_errAbort. No CPU fallback.
 */
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include "sonLib.h"
#include "pairwiseAligner.h"
#include "multipleAligner.h"
#include "stateMachine.h"
#include "barb200.h"
#include "barb200_shim_env.h"

/* defined in impl/pairwiseAligner.c:1222-1233 (not static) but missing from pairwiseAligner.h */
stList *getAnchorPairsForPairwiseAlignmentParameters(const char *sX, const char *sY, const int64_t lX, const int64_t lY,
                                                    PairwiseAlignmentParameters *p);

static pthread_mutex_t shim_mutex = PTHREAD_MUTEX_INITIALIZER;
static barb200_ctx *shim_ctx = NULL;

static barb200_ctx *shim_context(void) {
    pthread_mutex_lock(&shim_mutex);
    if (shim_ctx == NULL) {
        barb200_params p;
        char err[256];
        barb200_params_default(&p);                       /* the POA fields are not used by the pair-HMM path */
        barb200_devices_from_env(&p);                     /* BARB200_DEVICE / BARB200_DEVICES, as in POA mode */
        shim_ctx = barb200_create(&p, err, (int)sizeof(err));
        if (shim_ctx == NULL) {
            pthread_mutex_unlock(&shim_mutex);
            st_errAbort("barb200: cannot create the GPU engine: %s", err);
        }
    }
    pthread_mutex_unlock(&shim_mutex);
    return shim_ctx;
}

static void params_from_pecan(const PairwiseAlignmentParameters *p, barb200_pecan_params *q) {
    barb200_pecan_params_default(q);
    q->threshold = p->threshold;
    q->min_diags_between_traceback = p->minDiagsBetweenTraceBack;
    q->traceback_diagonals = p->traceBackDiagonals;
    q->diagonal_expansion = p->diagonalExpansion;
    q->split_matrix_bigger_than_this = p->splitMatrixBiggerThanThis;
    q->dynamic_anchor_expansion = p->dynamicAnchorExpansion;
}

/* The engine hard-codes the constants of stateMachine5_construct(fiveState) (stateMachine.c:482-521). StateMachine5's fields
 * are private to stateMachine.c, so a machine is verified through its public face: every (emission, transition) pair that
 * cellCalculate hands to its callback, for all 25 symbol pairs, and the start / end vectors must equal those of a freshly
 * constructed default machine -- a five-state machine loaded from a trained HMM (hmm_getStateMachine) is REJECTED, not
 * silently mis-evaluated. Verified once per machine. */
typedef struct { double v[64]; int n; } sm_probe;
static void probe_transition(double *from, double *to, int64_t f, int64_t t, double eP, double tP, void *extra) {
    sm_probe *q = extra;
    (void)from; (void)to;
    if (q->n + 4 <= 64) { q->v[q->n++] = (double)f; q->v[q->n++] = (double)t; q->v[q->n++] = eP; q->v[q->n++] = tP; }
}
static void check_state_machine(StateMachine *sM) {
    static StateMachine *verified = NULL;
    if (sM->type != fiveState) st_errAbort("barb200: only the five-state pair-HMM (stateMachine5_construct(fiveState)) is supported");
    pthread_mutex_lock(&shim_mutex);
    const int known = sM == verified;
    pthread_mutex_unlock(&shim_mutex);
    if (known) return;
    StateMachine *d = stateMachine5_construct(fiveState);
    int same = sM->stateNumber == d->stateNumber;
    double cells[20];
    memset(cells, 0, sizeof(cells));
    for (int cx = 0; cx < SYMBOL_NUMBER && same; cx++) {
        for (int cy = 0; cy < SYMBOL_NUMBER && same; cy++) {
            sm_probe a, b;
            memset(&a, 0, sizeof(a)); memset(&b, 0, sizeof(b));
            sM->cellCalculate(sM, cells, cells + 5, cells + 10, cells + 15, (Symbol)cx, (Symbol)cy, probe_transition, &a);
            d->cellCalculate(d, cells, cells + 5, cells + 10, cells + 15, (Symbol)cx, (Symbol)cy, probe_transition, &b);
            same = a.n == b.n && memcmp(a.v, b.v, sizeof(double) * (size_t)a.n) == 0;
        }
    }
    for (int64_t st = 0; st < d->stateNumber && same; st++) {
        same = sM->startStateProb(sM, st) == d->startStateProb(d, st) && sM->endStateProb(sM, st) == d->endStateProb(d, st) &&
               sM->raggedStartStateProb(sM, st) == d->raggedStartStateProb(d, st) && sM->raggedEndStateProb(sM, st) == d->raggedEndStateProb(d, st);
    }
    stateMachine_destruct(d);
    if (!same) st_errAbort("barb200: the pair-HMM's transition / emission constants differ from stateMachine5_construct(fiveState); "
                           "trained HMMs are not supported by the GPU engine");
    pthread_mutex_lock(&shim_mutex);
    verified = sM;
    pthread_mutex_unlock(&shim_mutex);
}

static int64_t *flatten_anchors(stList *anchorPairs, int64_t *n) {
    *n = stList_length(anchorPairs);
    int64_t *a = st_malloc(sizeof(int64_t) * 2 * (*n > 0 ? *n : 1));
    for (int64_t i = 0; i < *n; i++) {
        stIntTuple *t = stList_get(anchorPairs, i);
        a[2 * i] = stIntTuple_get(t, 0);
        a[2 * i + 1] = stIntTuple_get(t, 1);
    }
    return a;
}

static stList *triples_to_list(int64_t *trip, int64_t n) {
    stList *l = stList_construct3(0, (void (*)(void *)) stIntTuple_destruct);
    for (int64_t i = 0; i < n; i++) {
        stList_append(l, stIntTuple_construct3(trip[3 * i], trip[3 * i + 1], trip[3 * i + 2]));
    }
    return l;
}

stList *getAlignedPairsUsingAnchors(StateMachine *sM, const char *sX, const char *sY, stList *anchorPairs, PairwiseAlignmentParameters *p,
                                    bool alignmentHasRaggedLeftEnd, bool alignmentHasRaggedRightEnd) {
    check_state_machine(sM);
    barb200_ctx *ctx = shim_context();
    barb200_pecan_params q;
    params_from_pecan(p, &q);
    int64_t lX = strlen(sX), lY = strlen(sY), nA, nOut = 0, *trip = NULL;
    int64_t *anchors = flatten_anchors(anchorPairs, &nA);
    const int64_t *ap = anchors;
    uint8_t rl = alignmentHasRaggedLeftEnd, rr = alignmentHasRaggedRightEnd;
    if (barb200_pecan_aligned_pairs_batch(ctx, &q, 1, &sX, &lX, &sY, &lY, &ap, &nA, &rl, &rr, &trip, &nOut, NULL, NULL) != BARB200_OK) {
        st_errAbort("barb200: pair-HMM batch failed: %s", barb200_last_error(ctx));
    }
    stList *alignedPairs = triples_to_list(trip, nOut);
    barb200_free(trip);
    free(anchors);
    return alignedPairs;
}

/* getAlignmentScore, multipleAligner.c:603-617 (static there) */
static int64_t alignment_score(int64_t *trip, int64_t n, int64_t seqLength1, int64_t seqLength2) {
    int64_t alignmentScore = 0;
    for (int64_t i = 0; i < n; i++) {
        alignmentScore += trip[3 * i];
    }
    int64_t j = seqLength1 < seqLength2 ? seqLength1 : seqLength2;
    j = j == 0 ? 1 : j;
    double d = (double) alignmentScore / (j * PAIR_ALIGNMENT_PROB_1);
    d = d > 1.0 ? 1.0 : d;
    d = d < 0.0 ? 0.0 : d;
    return d * PAIR_ALIGNMENT_PROB_1;
}

/* addMultipleAlignedPairs (multipleAligner.c:651-666, static there) for a LIST of sequence pairs in one device batch: pair i is
 * (first[i], second[i]); the pairs' 5-tuples are appended to multipleAlignedPairs and (similarity, first, second) to scores, pair
 * after pair in list order -- exactly what the reference's one-pair-at-a-time loop leaves behind. */
static void align_pair_list(StateMachine *sM, stList *seqFrags, const int64_t *first, const int64_t *second, int64_t pairNo,
                            PairwiseAlignmentParameters *p, stList *multipleAlignedPairs, stList *scores) {
    if (pairNo <= 0) {
        return;
    }
    check_state_machine(sM);
    barb200_ctx *ctx = shim_context();
    barb200_pecan_params q;
    params_from_pecan(p, &q);
    const char **sx = st_malloc(sizeof(char *) * pairNo), **sy = st_malloc(sizeof(char *) * pairNo);
    int64_t *lx = st_malloc(8 * pairNo), *ly = st_malloc(8 * pairNo), *na = st_malloc(8 * pairNo), *nOut = st_malloc(8 * pairNo);
    int64_t **anchors = st_malloc(sizeof(int64_t *) * pairNo), **trip = st_malloc(sizeof(int64_t *) * pairNo);
    uint8_t *rl = st_malloc(pairNo), *rr = st_malloc(pairNo);
    for (int64_t i = 0; i < pairNo; i++) {
        SeqFrag *f1 = stList_get(seqFrags, first[i]), *f2 = stList_get(seqFrags, second[i]);
        sx[i] = f1->seq; sy[i] = f2->seq; lx[i] = strlen(f1->seq); ly[i] = strlen(f2->seq);
        rl[i] = f1->leftEndId != f2->leftEndId;                /* addMultipleAlignedPairs, multipleAligner.c:660-661 */
        rr[i] = f1->rightEndId != f2->rightEndId;
    }
    /* anchors (getAlignedPairs, pairwiseAligner.c:1527-1534): MUM chains of the whole round in one device batch. A pair with
     * lX * lY <= anchorMatrixBiggerThanThis has no anchors (:1224-1226), so a round of such pairs (short ends, the common case)
     * makes no anchor call at all. */
    if (p->useMumAnchors) {
        int64_t searched = 0;
        for (int64_t i = 0; i < pairNo; i++) {
            anchors[i] = NULL; na[i] = 0;
            searched += lx[i] * ly[i] > p->anchorMatrixBiggerThanThis;
        }
        barb200_mum_params mp;
        mp.k = p->k; mp.u = p->u; mp.anchor_matrix_bigger_than_this = p->anchorMatrixBiggerThanThis; mp.recursive_mums = (int)p->recursiveMums;
        if (searched > 0 && barb200_pecan_anchor_pairs_batch(ctx, &mp, pairNo, sx, lx, sy, ly, anchors, na) != BARB200_OK) {
            st_errAbort("barb200: MUM anchor batch failed: %s", barb200_last_error(ctx));
        }
    } else {
        /* the lastz path: the reference's host code, one pair per thread -- the reference itself runs it concurrently from
         * bar()'s OpenMP loop over ends (bar/impl/bar.c:90-94) */
#if defined(_OPENMP)
#pragma omp parallel for schedule(dynamic, 1)
#endif
        for (int64_t i = 0; i < pairNo; i++) {
            stList *anchorPairs = getAnchorPairsForPairwiseAlignmentParameters(sx[i], sy[i], lx[i], ly[i], p);
            anchors[i] = flatten_anchors(anchorPairs, &na[i]);
            stList_destruct(anchorPairs);
        }
    }
    if (barb200_pecan_aligned_pairs_batch(ctx, &q, pairNo, sx, lx, sy, ly, (const int64_t *const *) anchors, na, rl, rr, trip, nOut, NULL, NULL) != BARB200_OK) {
        st_errAbort("barb200: pair-HMM batch failed: %s", barb200_last_error(ctx));
    }
    for (int64_t k = 0; k < pairNo; k++) {
        SeqFrag *f1 = stList_get(seqFrags, first[k]), *f2 = stList_get(seqFrags, second[k]);
        stList *alignedPairs = reweightAlignedPairs2(triples_to_list(trip[k], nOut[k]), f1->length, f2->length, p->gapGamma);
        int64_t distance;
        if (p->gapGamma <= 0.0) {
            distance = alignment_score(trip[k], nOut[k], f1->length, f2->length);
        } else {                                           /* scores were reweighted: sum them from the list */
            int64_t n = stList_length(alignedPairs), *t2 = st_malloc(24 * (n > 0 ? n : 1));
            for (int64_t i = 0; i < n; i++) { t2[3 * i] = stIntTuple_get(stList_get(alignedPairs, i), 0); }
            distance = alignment_score(t2, n, f1->length, f2->length);
            free(t2);
        }
        /* convertAlignedPairsToMultipleAlignedPairs, multipleAligner.c:619-633 (static there): pops, i.e. reverses */
        while (stList_length(alignedPairs) > 0) {
            stIntTuple *aP = stList_pop(alignedPairs);
            stList_append(multipleAlignedPairs, stIntTuple_construct5(stIntTuple_get(aP, 0), first[k], stIntTuple_get(aP, 1), second[k], stIntTuple_get(aP, 2)));
            stIntTuple_destruct(aP);
        }
        stList_destruct(alignedPairs);
        stList_append(scores, stIntTuple_construct3(distance, first[k], second[k]));
        barb200_free(trip[k]);
        free(anchors[k]);                                  /* malloc'd by either path (barb200_free is free), or NULL */
    }
    free(sx); free(sy); free(lx); free(ly); free(na); free(nOut); free(anchors); free(trip); free(rl); free(rr);
}

stList *makeAllPairwiseAlignments(StateMachine *sM, stList *seqFrags, PairwiseAlignmentParameters *p, stList **seqPairSimilarityScores) {
    *seqPairSimilarityScores = stList_construct3(0, (void (*)(void *)) stIntTuple_destruct);
    stList *multipleAlignedPairs = stList_construct3(0, (void (*)(void *)) stIntTuple_destruct);
    const int64_t seqNo = stList_length(seqFrags), pairNo = seqNo * (seqNo - 1) / 2;
    if (pairNo <= 0) {
        return multipleAlignedPairs;
    }
    int64_t *first = st_malloc(8 * pairNo), *second = st_malloc(8 * pairNo);
    int64_t k = 0;
    for (int64_t seq1 = 0; seq1 < seqNo; seq1++) {            /* the pairs in the reference's order, multipleAligner.c:675-679 */
        for (int64_t seq2 = seq1 + 1; seq2 < seqNo; seq2++, k++) {
            first[k] = seq1; second[k] = seq2;
        }
    }
    align_pair_list(sM, seqFrags, first, second, pairNo, p, multipleAlignedPairs, *seqPairSimilarityScores);
    free(first); free(second);
    return multipleAlignedPairs;
}

/* defined (not static) in multipleAligner.c but missing from multipleAligner.h */
stSortedSet *getReferencePairwiseAlignments2(stList *seqFrags);
int64_t *getDistanceMatrix(stSet *columns, stList *seqFrags, int64_t maxPairsToConsider);
int64_t getNextBestPair(int64_t seq1, int64_t *distanceCounts, int64_t seqNo, stSortedSet *chosenPairsOfSequencesToAlign);
stSet *getMultipleSequenceAlignment(stList *seqFrags, stList *multipleAlignedPairs, double gapGamma);
stSet *getMultipleSequenceAlignmentProgressive(stList *seqFrags, stList *multipleAlignedPairs, double gapGamma, stList *seqPairSimilarityScores);
stList *filterMultipleAlignedPairs(stSet *columns, stList *multipleAlignedPairs);

/* makeAlignment (inc/multipleAligner.h, impl/multipleAligner.c:887-939) -- the entry point of endAligner.c:87 (makeEndAlignment) and with
 * it of flowerAligner.c / bar() in the cPecan configuration. With fewer than all pairs affordable (spanningTrees * (n-1) < n(n-1)/2) the
 * reference aligns n-1 "reference" pairs and then, spanningTrees-1 times, one more pair per sequence chosen from the current MSA. WHICH
 * pairs are chosen in a round depends on the MSA of the previous round and on the pairs chosen so far -- not on the alignments of the
 * round itself -- so every round is selected first (same calls, same order, same st_random() draws as the reference's loop) and then
 * aligned as ONE device batch; the tuples are appended in the order the reference's one-by-one loop appends them. */
MultipleAlignment *makeAlignment(StateMachine *sM, stList *seqFrags, int64_t spanningTrees, int64_t maxPairsToConsider, bool useProgressiveMerging,
                                 float matchGamma, PairwiseAlignmentParameters *p) {
    int64_t seqNo = stList_length(seqFrags);
    if (spanningTrees * (seqNo - 1) >= (seqNo * (seqNo - 1)) / 2) {          /* all pairs: the reference's code, batched by makeAllPairwiseAlignments above */
        return makeAlignmentUsingAllPairs(sM, seqFrags, useProgressiveMerging, matchGamma, p);
    }
    MultipleAlignment *mA = st_calloc(1, sizeof(MultipleAlignment));
    mA->alignedPairs = stList_construct3(0, (void (*)(void *)) stIntTuple_destruct);
    mA->chosenPairwiseAlignments = stList_construct3(0, (void (*)(void *)) stIntTuple_destruct);
    stSortedSet *chosen = getReferencePairwiseAlignments2(seqFrags);
    int64_t cap = stSortedSet_size(chosen) + seqNo + 1, n = 0;
    int64_t *first = st_malloc(8 * cap), *second = st_malloc(8 * cap);
    stSortedSetIterator *pairIt = stSortedSet_getIterator(chosen);
    stIntTuple *pairToAlign;
    while ((pairToAlign = stSortedSet_getNext(pairIt)) != NULL) {           /* :898-906 */
        first[n] = stIntTuple_get(pairToAlign, 0); second[n] = stIntTuple_get(pairToAlign, 1); n++;
    }
    stSortedSet_destructIterator(pairIt);
    align_pair_list(sM, seqFrags, first, second, n, p, mA->alignedPairs, mA->chosenPairwiseAlignments);
    int64_t iteration = 0;
    while (1) {                                                              /* :910-937 */
        mA->columns = (stList_length(seqFrags) == 2 || useProgressiveMerging)
                ? getMultipleSequenceAlignmentProgressive(seqFrags, mA->alignedPairs, matchGamma, mA->chosenPairwiseAlignments)
                : getMultipleSequenceAlignment(seqFrags, mA->alignedPairs, matchGamma);
        if (++iteration >= spanningTrees) {
            stSortedSet_destruct(chosen);
            mA->alignedPairs = filterMultipleAlignedPairs(mA->columns, mA->alignedPairs);
            free(first); free(second);
            return mA;
        }
        int64_t *distanceCounts = getDistanceMatrix(mA->columns, seqFrags, maxPairsToConsider);
        stSet_destruct(mA->columns);
        n = 0;
        for (int64_t seq = 0; seq < seqNo; seq++) {                          /* selection: as the reference, the chosen set grows pair by pair */
            int64_t otherSeq = getNextBestPair(seq, distanceCounts, seqNo, chosen);
            if (otherSeq != INT64_MAX) {
                assert(seq != otherSeq);
                first[n] = seq; second[n] = otherSeq; n++;
                stSortedSet_insert(chosen, seq < otherSeq ? stIntTuple_construct2(seq, otherSeq) : stIntTuple_construct2(otherSeq, seq));
            }
        }
        free(distanceCounts);
        align_pair_list(sM, seqFrags, first, second, n, p, mA->alignedPairs, mA->chosenPairwiseAlignments);
    }
    return NULL;
}
