/*
 * end_trace_ref_harness.c -- TEST INFRASTRUCTURE ONLY. The window chain of the UNMODIFIED reference msa_make_partial_order_alignment
 * (bar/impl/poaBarAligner.c:463-749, its own compiled object), observed from outside and returned in barb200_trace_ends' word
 * layout (include/barb200.h). end_trace.mk links poaBarAligner.o with
 *   -Wl,--wrap=abpoa_msa        every window's job: its lengths, codes and progressive flag as the reference's loop made them; the
 *                               same job is traced through ref_harness.c:ref_poa_msa_trace (abPOA's own per-alignment state), and
 *                               then the reference's abpoa_msa runs as it would have; its MSA must equal the trace's
 *   -Wl,--wrap=st_calloc        the loop's first two allocations are its seq_offsets and empty_seqs arrays (:494-497): the
 *                               offsets and N stand-in flags at each abpoa_msa call are read from the reference's own variables
 *   -Wl,--wrap=stList_append / stList_destruct
 *                               the windows it keeps (:692), read just before it frees them (:743): their row lengths and columns
 *                               after the trims, as its stitch used them
 * Nothing is recorded outside bar_trace_ref_ends' own msa_make_partial_order_alignment calls, so the wrapped entry points of
 * bar_ref_harness.c (included below) compute exactly what libbar_ref.so computes.
 */
#include <stdbool.h>
#include "bar_ref_harness.c"

int64_t *ref_poa_msa_trace(const ref_params_t *p, int n_seq, const int *lens, const uint8_t *flat, int64_t *n_words);

typedef struct { int64_t *w; size_t n, m; } rbuf_t;
static void rpush(rbuf_t *b, int64_t v) {
    if (b->n == b->m) { b->m = b->m ? b->m * 2 : 1024; b->w = (int64_t *)realloc(b->w, b->m * sizeof(int64_t)); }
    b->w[b->n++] = v;
}

/* the state of one observed msa_make_partial_order_alignment call (thread-local: the reference may run ends in parallel) */
static __thread int armed, inside, n_calloc, failed;
static __thread int64_t cur_seq_no, n_win;
static __thread const ref_params_t *cur_p;
static __thread rbuf_t *cur_buf;
static __thread int64_t *cur_offsets;
static __thread bool *cur_empty;
static __thread stList *cur_windows;
static __thread size_t *trim_at;                 /* where each window's trimmed lengths go in cur_buf */
static __thread int64_t trim_cap;
static __thread int trim_read;

void *__real_st_calloc(int64_t n, size_t size);
void *__wrap_st_calloc(int64_t n, size_t size) {
    void *p = __real_st_calloc(n, size);
    if (armed && !inside && n_calloc < 2) {
        if (n != cur_seq_no || size != (n_calloc == 0 ? sizeof(int64_t) : sizeof(bool))) failed = 1;   /* the loop has changed */
        if (n_calloc == 0) cur_offsets = (int64_t *)p; else cur_empty = (bool *)p;
        ++n_calloc;
    }
    return p;
}

void __real_stList_append(stList *l, void *item);
void __wrap_stList_append(stList *l, void *item) {
    if (armed && !inside && !cur_windows) cur_windows = l;
    __real_stList_append(l, item);
}

void __real_stList_destruct(stList *l);
void __wrap_stList_destruct(stList *l) {
    if (armed && !inside && l == cur_windows && stList_length(l) == n_win) {
        for (int64_t k = 0; k < n_win; ++k) {
            Msa *m = (Msa *)stList_get(l, k);
            for (int64_t i = 0; i < cur_seq_no; ++i) cur_buf->w[trim_at[k] + i] = m->seq_lens[i];
            cur_buf->w[trim_at[k] + cur_seq_no] = m->column_no;
        }
        trim_read = 1;
    }
    __real_stList_destruct(l);
}

int __real_abpoa_msa(abpoa_t *ab, abpoa_para_t *abpt, int n_seqs, char **seq_names, int *seq_lens, uint8_t **seqs, int **qual_weights,
                     FILE *out_fp);
int __wrap_abpoa_msa(abpoa_t *ab, abpoa_para_t *abpt, int n_seqs, char **seq_names, int *seq_lens, uint8_t **seqs, int **qual_weights,
                     FILE *out_fp) {
    if (!armed || inside) return __real_abpoa_msa(ab, abpt, n_seqs, seq_names, seq_lens, seqs, qual_weights, out_fp);
    inside = 1;
    rbuf_t *b = cur_buf;
    if (n_seqs != cur_seq_no || n_calloc < 2) failed = 1;
    if (n_win == trim_cap) { trim_cap = trim_cap ? 2 * trim_cap : 64; trim_at = (size_t *)realloc(trim_at, sizeof(size_t) * trim_cap); }
    rpush(b, n_win);
    for (int i = 0; i < n_seqs; ++i) rpush(b, cur_offsets ? cur_offsets[i] : -1);
    for (int i = 0; i < n_seqs; ++i) rpush(b, seq_lens[i]);
    for (int i = 0; i < n_seqs; ++i) rpush(b, cur_empty ? cur_empty[i] : -1);
    rpush(b, abpt->progressive_poa);
    size_t tot = 0;
    for (int i = 0; i < n_seqs; ++i) tot += seq_lens[i];
    uint8_t *flat = (uint8_t *)malloc(tot > 0 ? tot : 1);
    for (int i = 0, o = 0; i < n_seqs; o += seq_lens[i], ++i) memcpy(flat + o, seqs[i], seq_lens[i]);
    ref_params_t q = *cur_p;
    q.progressive_poa = abpt->progressive_poa;
    int64_t nw = 0;
    int64_t *tr = ref_poa_msa_trace(&q, n_seqs, seq_lens, flat, &nw);
    rpush(b, nw);
    for (int64_t k = 0; k < nw; ++k) rpush(b, tr[k]);
    trim_at[n_win++] = b->n;
    for (int i = 0; i <= n_seqs; ++i) rpush(b, 0);
    const int rc = __real_abpoa_msa(ab, abpt, n_seqs, seq_names, seq_lens, seqs, qual_weights, out_fp);
    /* the trace is of the job the reference ran: its MSA is the one the reference goes on with */
    const int ml = (int)tr[1];
    const size_t nwm = ((size_t)n_seqs * ml + 7) / 8;
    const uint8_t *tm = (const uint8_t *)(tr + (nw - (int64_t)nwm));
    if (ab->abc->msa_len != ml) failed = 1;
    else for (int i = 0; i < n_seqs; ++i) if (memcmp(ab->abc->msa_base[i], tm + (size_t)i * ml, ml)) failed = 1;
    free(tr); free(flat);
    inside = 0;
    return rc;
}

static void push_msa(rbuf_t *b, int64_t seq_no, int64_t cols, const uint8_t *flat) {
    const size_t nb = (size_t)seq_no * cols, nwm = (nb + 7) / 8;
    rpush(b, seq_no); rpush(b, cols);
    const size_t at = b->n;
    for (size_t k = 0; k < nwm; ++k) rpush(b, 0);
    memcpy(b->w + at, flat, nb);
}

/* barb200_trace_ends' layout for every end from the reference's own loop; right_end_indexes == NULL: independent ends. Returns 0,
 * or -1 when the observation failed (the reference's loop no longer matches what the wraps expect, or a trace's MSA differs from
 * the reference's window MSA); then no arrays are left. */
int bar_trace_ref_ends(const ref_params_t *p, int64_t end_no, int64_t *end_lengths, char ***end_strings, int **end_string_lengths,
                       int64_t **right_end_indexes, int64_t **right_end_row_indexes, int64_t **overlaps, int64_t window_size,
                       int64_t max_prog_rows, double max_prog_length_diff, int64_t **trace_out, int64_t *n_words) {
    abpoa_para_t *abpt = make_para(p);
    rbuf_t *bs = (rbuf_t *)calloc(end_no > 0 ? end_no : 1, sizeof(rbuf_t));
    int bad = 0;
    for (int64_t e = 0; e < end_no; ++e) {
        const int64_t K = end_lengths[e];
        rpush(&bs[e], K); rpush(&bs[e], 0);
        armed = 1; inside = 0; n_calloc = 0; failed = 0; trim_read = 0; n_win = 0;
        cur_seq_no = K; cur_p = p; cur_buf = &bs[e]; cur_offsets = NULL; cur_empty = NULL; cur_windows = NULL;
        Msa *m = msa_make_partial_order_alignment(dup_strings(end_strings[e], end_string_lengths[e], K), dup_ints(end_string_lengths[e], K),
                                                  K, window_size, max_prog_rows, max_prog_length_diff, abpt);
        armed = 0;
        bs[e].w[1] = n_win;
        if (n_win == 1 && !trim_read) {        /* a single window is returned as the output itself (:705-710) */
            for (int64_t i = 0; i < K; ++i) {
                int64_t n = 0;
                for (int64_t c = 0; c < m->column_no; ++c) n += m->msa_seq[i][c] != 5;
                bs[e].w[trim_at[0] + i] = n;
            }
            bs[e].w[trim_at[0] + K] = m->column_no;
        } else if (n_win > 1 && !trim_read) failed = 1;
        if (!right_end_indexes) { uint8_t *f = flatten(m); push_msa(&bs[e], K, m->column_no, f); free(f); }
        msa_destruct(m);
        bad |= failed;
    }
    if (right_end_indexes && !bad) {
        int64_t *cols = (int64_t *)malloc(sizeof(int64_t) * (end_no > 0 ? end_no : 1));
        uint8_t **outs = (uint8_t **)malloc(sizeof(uint8_t *) * (end_no > 0 ? end_no : 1));
        bar_ref_make_consistent_partial_order_alignments(p, end_no, end_lengths, end_strings, end_string_lengths, right_end_indexes,
                                                         right_end_row_indexes, overlaps, window_size, max_prog_rows, max_prog_length_diff,
                                                         cols, outs);
        for (int64_t e = 0; e < end_no; ++e) { push_msa(&bs[e], end_lengths[e], cols[e], outs[e]); free(outs[e]); }
        free(cols); free(outs);
    }
    abpoa_free_para(abpt);
    for (int64_t e = 0; e < end_no; ++e) {
        if (bad) { free(bs[e].w); trace_out[e] = NULL; n_words[e] = 0; }
        else { trace_out[e] = bs[e].w; n_words[e] = (int64_t)bs[e].n; }
    }
    free(bs);
    return bad ? -1 : 0;
}
