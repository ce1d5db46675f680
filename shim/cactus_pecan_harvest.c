/*
 * cactus_pecan_harvest.c -- instrumentation for a REFERENCE (CPU) Cactus build in the cPecan configuration
 * (bar/partialOrderAlignment="0"): records every sequence pair cPecan's multiple aligner aligns during a bar() run, with its
 * parameters, the reference's anchors and hashes of the reference's results, so that the pair-HMM / MUM-anchor workload of a real
 * dataset (10way-MHC, BASELINE.json configs[3]; the data is not available offline) can be captured once on a box that has it and
 * replayed anywhere by scripts/pecan_replay.py (workload.read_pecan_harvest), parity-checked pair by pair.
 *
 * Build hook (oracle/pecan_harvest.mk does exactly this for oracle/_ref/libflower_pecan_harvest.so), the recipe of
 * shim/cactus_bar_harvest.c applied to cPecan's two objects: pairwiseAligner.o and multipleAligner.o are each linked TWICE --
 * once with the wrapped entry point weakened (getAlignedPairs resp. makeAlignment; every caller in another object reaches the
 * wrapper below), once as a private copy whose global symbols carry the prefix ref_, which the wrappers forward to:
 *     objcopy --weaken-symbol=getAlignedPairs pairwiseAligner.o pairwiseAligner_weak.o
 *     objcopy --weaken-symbol=makeAlignment multipleAligner.o multipleAligner_weak.o
 *     nm -g --defined-only X.o | awk '{print $3 " ref_" $3}' > syms;  objcopy --redefine-syms=syms X.o X_private.o
 * Both wrapped calls cross object files: addMultipleAlignedPairs (multipleAligner.c:651-666) calls getAlignedPairs
 * (pairwiseAligner.c:1527-1534) once per chosen pair, and makeEndAlignment (endAligner.c:87) calls makeAlignment
 * (multipleAligner.c:887-939) once per end. The private makeAlignment's own getAlignedPairs calls are undefined in its object, so
 * they reach the wrapper too. The alignment itself is the unmodified reference's.
 *
 * Recording: with BARB200_PECAN_HARVEST=<path> set, every getAlignedPairs call appends one record, under a mutex. Pairs are grouped
 * by end: makeAlignment takes the next end id (0, 1, 2, ... in the order the calls start) and the pairs its thread aligns until it
 * returns are numbered 0, 1, 2, ... within that end (bar() aligns ends concurrently; the id is thread-local). A pair aligned
 * outside any makeAlignment has end id -1. Without the variable the wrappers only forward (and count, pecan_harvest_pair_calls).
 *
 * Record layout (little endian; i64 = int64, u64 = uint64, f64 = double):
 *   i64 magic 0x484E435032303042 ("B002PCNH")
 *   i64 end_id, pair_index
 *   f64 threshold
 *   i64 minDiagsBetweenTraceBack, traceBackDiagonals, diagonalExpansion, splitMatrixBiggerThanThis, dynamicAnchorExpansion,
 *       anchorMatrixBiggerThanThis, k, u, recursiveMums, useMumAnchors, raggedLeft, raggedRight
 *   i64 lX, lY, n_anchors
 *   u64 anchor_hash; i64 n_triples; u64 triple_hash
 *   lX bytes sX, lY bytes sY
 *   n_anchors x (i64 x, i64 y): the anchors of getAnchorPairsForPairwiseAlignmentParameters (pairwiseAligner.c:1222-1231)
 * anchor_hash is the 64-bit FNV-1a (offset basis 0xcbf29ce484222325, prime 0x100000001b3) over the anchors' 16 * n_anchors bytes
 * as written above; triple_hash the same over the 24 * n_triples bytes of the returned (score, x, y) triples, in the order
 * getAlignedPairs returns them.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "sonLib.h"
#include "pairwiseAligner.h"
#include "multipleAligner.h"

#define PECAN_HARVEST_MAGIC 0x484E435032303042LL

stList *ref_getAlignedPairs(StateMachine *sM, const char *sX, const char *sY, PairwiseAlignmentParameters *p, bool alignmentHasRaggedLeftEnd,
                            bool alignmentHasRaggedRightEnd);
MultipleAlignment *ref_makeAlignment(StateMachine *sM, stList *seqFrags, int64_t spanningTrees, int64_t maxPairsToConsider,
                                     bool useProgressiveMerging, float matchGamma, PairwiseAlignmentParameters *pairwiseAlignmentBandingParameters);
/* defined in impl/pairwiseAligner.c:1222-1233 (not static) but missing from pairwiseAligner.h */
stList *getAnchorPairsForPairwiseAlignmentParameters(const char *sX, const char *sY, const int64_t lX, const int64_t lY,
                                                    PairwiseAlignmentParameters *p);

static pthread_mutex_t harvest_mutex = PTHREAD_MUTEX_INITIALIZER;
static int64_t next_end_id = 0, pair_calls = 0;
static __thread int64_t tl_end_id = -1, tl_pair_index = 0;

/* getAlignedPairs calls since the library was loaded, recorded or not (tests: records lost or duplicated under concurrency) */
int64_t pecan_harvest_pair_calls(void) {
    pthread_mutex_lock(&harvest_mutex);
    const int64_t n = pair_calls;
    pthread_mutex_unlock(&harvest_mutex);
    return n;
}

static uint64_t fnv1a(uint64_t h, const void *data, size_t n) {
    const unsigned char *b = data;
    for (size_t i = 0; i < n; i++) {
        h ^= b[i];
        h *= 0x100000001b3ULL;
    }
    return h;
}

static uint64_t hash_tuples(stList *l, int64_t width) {
    uint64_t h = 0xcbf29ce484222325ULL;
    for (int64_t i = 0; i < stList_length(l); i++) {
        stIntTuple *t = stList_get(l, i);
        for (int64_t k = 0; k < width; k++) {
            const int64_t v = stIntTuple_get(t, k);
            h = fnv1a(h, &v, sizeof(v));
        }
    }
    return h;
}

static void put64(FILE *f, int64_t v) { fwrite(&v, sizeof(v), 1, f); }

static void harvest(int64_t end_id, int64_t pair_index, const char *sX, const char *sY, PairwiseAlignmentParameters *p, bool raggedLeft,
                    bool raggedRight, stList *alignedPairs) {
    const char *path = getenv("BARB200_PECAN_HARVEST");
    if (path == NULL) return;
    const int64_t lX = strlen(sX), lY = strlen(sY);
    stList *anchorPairs = getAnchorPairsForPairwiseAlignmentParameters(sX, sY, lX, lY, p);
    const int64_t nA = stList_length(anchorPairs);
    const uint64_t anchor_hash = hash_tuples(anchorPairs, 2), triple_hash = hash_tuples(alignedPairs, 3);
    pthread_mutex_lock(&harvest_mutex);
    FILE *f = fopen(path, "ab");
    if (f != NULL) {
        put64(f, PECAN_HARVEST_MAGIC); put64(f, end_id); put64(f, pair_index);
        fwrite(&p->threshold, sizeof(double), 1, f);
        put64(f, p->minDiagsBetweenTraceBack); put64(f, p->traceBackDiagonals); put64(f, p->diagonalExpansion);
        put64(f, p->splitMatrixBiggerThanThis); put64(f, p->dynamicAnchorExpansion); put64(f, p->anchorMatrixBiggerThanThis);
        put64(f, p->k); put64(f, p->u); put64(f, p->recursiveMums); put64(f, p->useMumAnchors); put64(f, raggedLeft); put64(f, raggedRight);
        put64(f, lX); put64(f, lY); put64(f, nA);
        put64(f, (int64_t)anchor_hash); put64(f, stList_length(alignedPairs)); put64(f, (int64_t)triple_hash);
        fwrite(sX, 1, (size_t)lX, f);
        fwrite(sY, 1, (size_t)lY, f);
        for (int64_t i = 0; i < nA; i++) {
            stIntTuple *t = stList_get(anchorPairs, i);
            put64(f, stIntTuple_get(t, 0)); put64(f, stIntTuple_get(t, 1));
        }
        fclose(f);
    }
    pthread_mutex_unlock(&harvest_mutex);
    stList_destruct(anchorPairs);
}

stList *getAlignedPairs(StateMachine *sM, const char *sX, const char *sY, PairwiseAlignmentParameters *p, bool alignmentHasRaggedLeftEnd,
                        bool alignmentHasRaggedRightEnd) {
    const int64_t pair_index = tl_pair_index++;
    pthread_mutex_lock(&harvest_mutex);
    pair_calls++;
    pthread_mutex_unlock(&harvest_mutex);
    stList *alignedPairs = ref_getAlignedPairs(sM, sX, sY, p, alignmentHasRaggedLeftEnd, alignmentHasRaggedRightEnd);
    harvest(tl_end_id, pair_index, sX, sY, p, alignmentHasRaggedLeftEnd, alignmentHasRaggedRightEnd, alignedPairs);
    return alignedPairs;
}

MultipleAlignment *makeAlignment(StateMachine *sM, stList *seqFrags, int64_t spanningTrees, int64_t maxPairsToConsider,
                                 bool useProgressiveMerging, float matchGamma, PairwiseAlignmentParameters *pairwiseAlignmentBandingParameters) {
    const int64_t outer_end = tl_end_id, outer_index = tl_pair_index;
    pthread_mutex_lock(&harvest_mutex);
    tl_end_id = next_end_id++;
    pthread_mutex_unlock(&harvest_mutex);
    tl_pair_index = 0;
    MultipleAlignment *mA = ref_makeAlignment(sM, seqFrags, spanningTrees, maxPairsToConsider, useProgressiveMerging, matchGamma,
                                              pairwiseAlignmentBandingParameters);
    tl_end_id = outer_end;
    tl_pair_index = outer_index;
    return mA;
}
