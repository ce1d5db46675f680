/*
 * mum_oracle.c -- TEST INFRASTRUCTURE ONLY. Plain-C restatement of cPecan's MUM anchoring, the anchors Cactus' BAR phase
 * computes for every sequence pair in cPecan mode (partialOrderAlignment="0", useMumAnchors="1"). Nothing in the product
 * may link or call this file; tests/ use it as the checker of K5 (cactus_b200/csrc/mum_anchor.cu) next to the compiled
 * reference (oracle/_ref/libmum_ref.so, oracle/mum_ref_harness.c) that pins it. Built by oracle/mum.mk.
 *
 * Paths relative to /root/reference/submodules/cPecan/impl.
 */
#include <ctype.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ---- getAnchorPairsForPairwiseAlignmentParameters with useMumAnchors = 1 (pairwiseAligner.c:1222-1231): maximal unique
 * matches, chained (getAlignedMums / getAlignedMums2 :2063-2121). Followed as written:
 *   cmpKmers (tolower bytes) :1848-1861, getSortedKmers :1873-1890, getMatchLength :1892-1899,
 *   getLongestUniqueMatch with the neighbour test against u :1905-1937, the MUM rule pXEnd < x || pDiag != x - y :2079-2080,
 *   updateSweepLine :1972-2008, chainMum :2014-2028, tracebackMums (one non-recursive level into every gap whose area exceeds
 *   anchorMatrixBiggerThanThis, reversal at the top level only) :2034-2061.
 * The sweep line (an stSortedSet keyed by end y, mum_sweep_cmp :1964-1967) is a plain array kept in that order; MUMs are
 * records in one array with the index of their predecessor. The list of MUMs waiting for their end x (mumsToAdd) keeps
 * creation order, as stList does. *would_abort is set when a MUM ends at lX: the reference's loops stop at lX - 1 and its
 * closing assert(stList_length(mumsToAdd) == 0) (:2113) fires in an assert-enabled build; without asserts that MUM is
 * simply never added, which is what this restatement does. ---------------------------------------------------------- */
typedef struct { int64_t k, u, bigger; int recursive; } mum_params_t;
typedef struct { int64_t x, y, length, score, pred; } omum_t;

static int cmp_kmers(const char *k1, const char *k2, int64_t k, int64_t *matchLength) {
    for (int64_t i = 0; i < k; i++) {
        if (tolower(k1[i]) < tolower(k2[i])) { *matchLength = i; return -1; }
        if (tolower(k1[i]) > tolower(k2[i])) { *matchLength = i; return 1; }
    }
    *matchLength = k;
    return 0;
}
static const char *g_sort_seq; static int64_t g_sort_k;
static int sort_kmers_cmp(const void *a, const void *b) {
    int64_t m;
    return cmp_kmers(g_sort_seq + *(const int64_t *)a, g_sort_seq + *(const int64_t *)b, g_sort_k, &m);
}
static int64_t match_length(const int64_t *sorted, int64_t n, const char *sY, const char *q, int64_t k, int64_t m) {
    if (m < 0 || m >= n) return 0;
    cmp_kmers(q, sY + sorted[m], k, &m);
    return m;
}
static int64_t longest_unique_match(const int64_t *sorted, int64_t n, const char *sY, const char *q, int64_t k, int64_t u, int64_t *ml) {
    int64_t l = 0, h = n, p = -2;
    *ml = 0;
    while (l < h) {
        int64_t m = (l + h) / 2, c;
        int i = cmp_kmers(q, sY + sorted[m], k, &c);
        if (c > *ml) { *ml = c; p = m; }
        if (i < 0) h = m; else if (i > 0) l = m + 1; else break;
    }
    return (*ml > u + match_length(sorted, n, sY, q, k, p - 1) && *ml > u + match_length(sorted, n, sY, q, k, p + 1)) ? p : -1;
}

typedef struct { int64_t *v; int64_t n, m; } ivec_t;
static void ipush(ivec_t *s, int64_t a) { if (s->n == s->m) { s->m = s->m ? 2 * s->m : 64; s->v = realloc(s->v, 8 * s->m); } s->v[s->n++] = a; }

static void aligned_mums2(const char *sX, const char *sY, int64_t lX, int64_t lY, const mum_params_t *p, int64_t oX, int64_t oY, int recursive,
                          ivec_t *out, int *would_abort, uint64_t *kmer_order_seed) {
    const int64_t k = p->k, ny = lY - k + 1;
    int64_t *sorted = NULL;
    if (ny > 0) {
        sorted = malloc(8 * ny);
        for (int64_t i = 0; i < ny; i++) sorted[i] = i;
        g_sort_seq = sY; g_sort_k = k;
        qsort(sorted, ny, 8, sort_kmers_cmp);
        if (kmer_order_seed && *kmer_order_seed) {        /* test aid: shuffle every run of equal k-mers */
            for (int64_t a = 0; a < ny;) {
                int64_t b = a + 1, m;
                while (b < ny && cmp_kmers(sY + sorted[a], sY + sorted[b], k, &m) == 0) b++;
                for (int64_t i = b - 1; i > a; i--) {
                    *kmer_order_seed = *kmer_order_seed * 6364136223846793005ULL + 1442695040888963407ULL;
                    int64_t j = a + (int64_t)((*kmer_order_seed >> 33) % (uint64_t)(i - a + 1)), t = sorted[i];
                    sorted[i] = sorted[j]; sorted[j] = t;
                }
                a = b;
            }
        }
    }
    const int64_t nx = lX - k + 1 > 0 ? lX - k + 1 : 0;
    omum_t *mums = malloc(sizeof(omum_t) * (nx > 0 ? nx : 1));
    int64_t n_mum = 0, *sweep = malloc(8 * (nx > 0 ? nx : 1)), n_sw = 0;
    ivec_t pend = {0};                                   /* mumsToAdd, creation order */
#define END_Y(i) (mums[i].y + mums[i].length)
    int64_t pDiag = -1, pXEnd = -1;
    for (int64_t x = 0; x < lX; x++) {
        /* updateSweepLine(x) */
        int64_t keep = 0;
        for (int64_t q = 0; q < pend.n; q++) {
            const int64_t i = pend.v[q];
            if (mums[i].x + mums[i].length != x) { pend.v[keep++] = i; continue; }
            int64_t le = -1;                             /* searchLessThanOrEqual */
            for (int64_t s = 0; s < n_sw; s++) if (END_Y(sweep[s]) <= END_Y(i)) le = s;
            if (le >= 0 && mums[sweep[le]].score >= mums[i].score) continue;
            for (;;) {                                   /* searchGreaterThanOrEqual, remove while score <= */
                int64_t ge = -1;
                for (int64_t s = 0; s < n_sw; s++) if (END_Y(sweep[s]) >= END_Y(i)) { ge = s; break; }
                if (ge < 0 || mums[sweep[ge]].score > mums[i].score) break;
                memmove(sweep + ge, sweep + ge + 1, 8 * (n_sw - ge - 1)); n_sw--;
            }
            int64_t at = 0;
            while (at < n_sw && END_Y(sweep[at]) < END_Y(i)) at++;
            memmove(sweep + at + 1, sweep + at, 8 * (n_sw - at)); sweep[at] = i; n_sw++;
        }
        pend.n = keep;
        if (x >= lX - k + 1) continue;
        int64_t ml, j = longest_unique_match(sorted, ny, sY, sX + x, k, p->u, &ml);
        if (j >= 0 && j < ny) {
            const int64_t y = sorted[j];
            if (pXEnd < x || pDiag != x - y) {
                omum_t *m = &mums[n_mum];
                m->x = x; m->y = y; m->length = ml; m->pred = -1;
                for (int64_t s = 0; s < n_sw; s++) if (END_Y(sweep[s]) < y) m->pred = sweep[s];   /* searchLessThan */
                m->score = m->pred >= 0 ? mums[m->pred].score + ml : ml;
                ipush(&pend, n_mum++);
                pDiag = x - y; pXEnd = x + ml;
            }
        }
    }
    if (pend.n && would_abort) *would_abort = 1;
#undef END_Y
    /* tracebackMums */
    int64_t i = n_sw ? sweep[n_sw - 1] : -1, cx = lX, cy = lY;
    const int64_t start = out->n;
    while (i >= 0) {
        const omum_t *m = &mums[i];
        if (recursive) {
            const int64_t a = m->x + m->length, b = m->y + m->length;
            if ((cx - a) * (cy - b) > p->bigger) aligned_mums2(sX + a, sY + b, cx - a, cy - b, p, oX + a, oY + b, 0, out, would_abort, kmer_order_seed);
        }
        for (int64_t q = m->length - 1; q >= 0; q--) { ipush(out, oX + m->x + q); ipush(out, oY + m->y + q); }
        cx = m->x; cy = m->y;
        i = m->pred;
    }
    if (recursive) {
        if (cx * cy > p->bigger) aligned_mums2(sX, sY, cx, cy, p, oX, oY, 0, out, would_abort, kmer_order_seed);
        for (int64_t a = start / 2, b = out->n / 2 - 1; a < b; a++, b--) {     /* stList_reverse on (x, y) tuples */
            int64_t tx = out->v[2 * a], ty = out->v[2 * a + 1];
            out->v[2 * a] = out->v[2 * b]; out->v[2 * a + 1] = out->v[2 * b + 1]; out->v[2 * b] = tx; out->v[2 * b + 1] = ty;
        }
    }
    free(sorted); free(mums); free(sweep); free(pend.v);
}

/* Returns the number of anchors; *out = malloc'd n x 2 (x, y) in the reference's order (release with oracle_mum_free).
 * kmer_order_seed != 0 shuffles every run of equal k-mers after the sort (the result must not change). */
int64_t oracle_mum_anchor_pairs(const char *sX, int64_t lX, const char *sY, int64_t lY, const mum_params_t *p, uint64_t kmer_order_seed,
                                int64_t **out, int *would_abort) {
    ivec_t v = {0};
    if (would_abort) *would_abort = 0;
    if (lX * lY > p->bigger) aligned_mums2(sX, sY, lX, lY, p, 0, 0, p->recursive, &v, would_abort, &kmer_order_seed);
    if (!v.v) v.v = malloc(16);
    *out = v.v;
    return v.n / 2;
}

void oracle_mum_free(void *p) { free(p); }
