/*
 * mum_ref_harness.c -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * Flat (pointer + size) driver around the UNMODIFIED reference cPecan MUM anchoring
 * (/root/reference/submodules/cPecan/impl/pairwiseAligner.c, compiled by oracle/Makefile from where it lies; this file is
 * linked against those objects by oracle/mum.mk into oracle/_ref/libmum_ref.so). The reference objects are built with
 * asserts on: getAlignedMums2's closing assert (pairwiseAligner.c:2111) aborts the process on inputs where a MUM ends at
 * lX, so callers check the input with oracle_mum_anchor_pairs (oracle/mum_oracle.c: would_abort) first.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "pairwiseAligner.h"

/* getAnchorPairsForPairwiseAlignmentParameters (pairwiseAligner.c:1222-1231) with useMumAnchors = 1 and the given k, u,
 * anchorMatrixBiggerThanThis and recursiveMums: the anchors as n x 2 (x, y) in the reference's order (malloc'd, release with
 * mum_ref_free). */
stList *getAnchorPairsForPairwiseAlignmentParameters(const char *sX, const char *sY, const int64_t lX, const int64_t lY,
                                                    PairwiseAlignmentParameters *p);
int64_t mum_ref_anchor_pairs(const char *sx, int64_t lx, const char *sy, int64_t ly, int64_t k, int64_t u, int64_t bigger, int recursive,
                                   int64_t **out) {
    PairwiseAlignmentParameters *p = pairwiseAlignmentBandingParameters_construct();
    p->useMumAnchors = 1; p->k = k; p->u = u; p->anchorMatrixBiggerThanThis = bigger; p->recursiveMums = recursive;
    char *cx = malloc(lx + 1), *cy = malloc(ly + 1);
    memcpy(cx, sx, lx); cx[lx] = 0; memcpy(cy, sy, ly); cy[ly] = 0;
    stList *a = getAnchorPairsForPairwiseAlignmentParameters(cx, cy, lx, ly, p);
    int64_t n = stList_length(a), *o = malloc(16 * (n > 0 ? n : 1));
    for (int64_t i = 0; i < n; ++i) { stIntTuple *t = stList_get(a, i); o[2 * i] = stIntTuple_get(t, 0); o[2 * i + 1] = stIntTuple_get(t, 1); }
    stList_destruct(a);
    free(cx); free(cy);
    pairwiseAlignmentBandingParameters_destruct(p);
    *out = o;
    return n;
}


void mum_ref_free(void *p) { free(p); }
