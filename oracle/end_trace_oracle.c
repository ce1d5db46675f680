/*
 * end_trace_oracle.c -- TEST INFRASTRUCTURE ONLY (see poa_oracle.h). oracle_trace_ends: the restated window chain and cross-end
 * trim of bar_oracle.c (msa_make_partial_order_alignment, poaBarAligner.c:463-749; make_consistent_partial_order_alignments,
 * :751-801) with every window's POA job run through poa_oracle.c's traced MSA, emitting the word layout of barb200_trace_ends
 * (include/barb200.h). It reuses bar_oracle.c's static steps (flip, trim, fix_trimmed, ...) by including that file, so the chain
 * here is the same restatement the BAR-level oracle tests pin against the reference.
 */
#include "bar_oracle.c"

typedef struct { int64_t *w; size_t n, m; } tbuf_t;
static void tpush(tbuf_t *b, int64_t v) {
    if (b->n == b->m) { b->m = b->m ? b->m * 2 : 1024; b->w = (int64_t *)realloc(b->w, b->m * sizeof(int64_t)); }
    b->w[b->n++] = v;
}

/* one end: the window chain with its records in *b (the header K, n_windows first); returns the stitched MSA */
static oracle_msa_t *trace_end(const oracle_params_t *p, char **seqs, const int *seq_lens, int64_t seq_no, int64_t window_size,
                               int64_t max_prog_rows, double max_prog_length_diff, tbuf_t *b) {
    oracle_msa_t *out = (oracle_msa_t *)calloc(1, sizeof(oracle_msa_t));
    out->seq_no = seq_no; out->seq_lens = (int *)malloc(sizeof(int) * (seq_no > 0 ? seq_no : 1));
    memcpy(out->seq_lens, seq_lens, sizeof(int) * seq_no);
    tpush(b, seq_no); tpush(b, 0);
    if (seq_no == 1) {                                         /* :471-483 */
        out->column_no = seq_lens[0];
        out->msa = (uint8_t *)malloc(out->column_no > 0 ? out->column_no : 1);
        for (int64_t i = 0; i < out->column_no; ++i) out->msa[i] = to_byte(seqs[0][i]);
        return out;
    }
    int64_t overlap_size = (int64_t)(0.5f * window_size);     /* :487-491 */
    if (overlap_size > 0) --overlap_size;
    int64_t bases_remaining = 0;
    int64_t *seq_offsets = (int64_t *)calloc(seq_no, sizeof(int64_t)), *row_overlaps = (int64_t *)calloc(seq_no, sizeof(int64_t));
    char *empty_seqs = (char *)calloc(seq_no, 1);
    for (int64_t i = 0; i < seq_no; ++i) bases_remaining += seq_lens[i];
    wmsa_t **windows = NULL; int64_t n_win = 0;
    size_t *trim_at = NULL;                                    /* where each window's trimmed lengths go in *b */
    wmsa_t *prev = NULL;
    while (bases_remaining > 0) {
        if (prev) {                                            /* :520-534 */
            for (int64_t i = 0; i < seq_no; ++i) {
                row_overlaps[i] = 0;
                for (int64_t j = prev->m.column_no - overlap_size; j < prev->m.column_no; ++j)
                    if (WAT(prev, i, j) != GAP) ++row_overlaps[i];
                seq_offsets[i] -= row_overlaps[i];
                bases_remaining += row_overlaps[i];
            }
        }
        wmsa_t *w = (wmsa_t *)calloc(1, sizeof(wmsa_t));
        w->m.seq_no = seq_no; w->m.seq_lens = (int *)malloc(sizeof(int) * seq_no);
        size_t tot = 0;
        for (int64_t i = 0; i < seq_no; ++i) {
            int64_t n = seq_lens[i] - seq_offsets[i]; if (n > window_size) n = window_size; if (n < 0) n = 0;
            w->m.seq_lens[i] = (int)n; tot += n > 0 ? n : 1;
        }
        uint8_t *flat = (uint8_t *)malloc(tot); int *lens = (int *)malloc(sizeof(int) * seq_no); size_t o = 0;
        int empty_count = 0;
        for (int64_t i = 0; i < seq_no; ++i) {                 /* :543-562 incl. the N stand-in for empty rows */
            if (w->m.seq_lens[i] == 0) { empty_seqs[i] = 1; w->m.seq_lens[i] = 1; flat[o] = to_byte('N'); ++empty_count; }
            else { empty_seqs[i] = 0; for (int j = 0; j < w->m.seq_lens[i]; ++j) flat[o + j] = to_byte(seqs[i][seq_offsets[i] + j]); }
            lens[i] = w->m.seq_lens[i]; o += lens[i];
        }
        oracle_params_t pp = *p;                               /* :567-571 */
        if (seq_no > max_prog_rows || (1. - (double)w->m.seq_lens[seq_no - 1] / (double)w->m.seq_lens[0] > max_prog_length_diff))
            pp.progressive_poa = 0;
        tpush(b, n_win);
        for (int64_t i = 0; i < seq_no; ++i) tpush(b, seq_offsets[i]);
        for (int64_t i = 0; i < seq_no; ++i) tpush(b, lens[i]);
        for (int64_t i = 0; i < seq_no; ++i) tpush(b, empty_seqs[i]);
        tpush(b, pp.progressive_poa);
        int64_t nw = 0;
        int64_t *tr = oracle_poa_msa_trace(&pp, (int)seq_no, lens, flat, &nw);
        tpush(b, nw);
        for (int64_t k = 0; k < nw; ++k) tpush(b, tr[k]);
        const int msa_len = (int)tr[1];
        const size_t nb = (size_t)seq_no * msa_len, nwm = (nb + 7) / 8;
        uint8_t *msa = (uint8_t *)malloc(nb > 0 ? nb : 1);
        memcpy(msa, (const uint8_t *)(tr + (nw - (int64_t)nwm)), nb);
        free(tr); free(flat); free(lens);
        trim_at = (size_t *)realloc(trim_at, sizeof(size_t) * (n_win + 1));
        trim_at[n_win] = b->n;
        for (int64_t i = 0; i <= seq_no; ++i) tpush(b, 0);
        w->m.msa = msa; w->m.column_no = msa_len; w->stride = msa_len;
        for (int64_t i = 0; i < seq_no && empty_count > 0; ++i) {   /* :631-644 */
            if (empty_seqs[i]) for (int64_t j = 0; j < w->m.column_no; ++j) if (normalise(WAT(w, i, j)) != GAP) {
                WAT(w, i, j) = GAP; --w->m.seq_lens[i]; --empty_count; break;
            }
        }
        for (int64_t i = 0; i < seq_no; ++i) {                 /* :654-663 */
            for (int64_t j = 0; j < w->m.column_no; ++j) WAT(w, i, j) = normalise(WAT(w, i, j));
            bases_remaining -= w->m.seq_lens[i];
            seq_offsets[i] += w->m.seq_lens[i];
        }
        if (prev) {                                            /* :668-689 */
            flip(w);
            float *pcs = column_scores(prev), *cs = column_scores(w);
            for (int64_t i = 0; i < seq_no; ++i) {
                int64_t ov = w->m.seq_lens[i] < row_overlaps[i] ? w->m.seq_lens[i] : row_overlaps[i];
                if (ov > 0) trim(i, w, cs, i, prev, pcs, ov);
            }
            fix_trimmed(w); fix_trimmed(prev);
            flip(w);
            free(pcs); free(cs);
        }
        windows = (wmsa_t **)realloc(windows, sizeof(wmsa_t *) * (n_win + 1));
        windows[n_win++] = w; prev = w;
    }
    b->w[1] = n_win;
    for (int64_t k = 0; k < n_win; ++k) {                      /* the lengths the stitch uses, after both neighbours' trims */
        for (int64_t i = 0; i < seq_no; ++i) b->w[trim_at[k] + i] = windows[k]->m.seq_lens[i];
        b->w[trim_at[k] + seq_no] = windows[k]->m.column_no;
    }
    out->column_no = 0;
    for (int64_t k = 0; k < n_win; ++k) out->column_no += windows[k]->m.column_no;
    out->msa = (uint8_t *)malloc((size_t)seq_no * (out->column_no > 0 ? out->column_no : 1));
    for (int64_t i = 0; i < seq_no; ++i) {                     /* :703-736 */
        int64_t o = 0;
        for (int64_t k = 0; k < n_win; ++k) for (int64_t c = 0; c < windows[k]->m.column_no; ++c) AT(out, i, o++) = WAT(windows[k], i, c);
    }
    for (int64_t k = 0; k < n_win; ++k) wmsa_free(windows[k]);
    free(windows); free(trim_at); free(seq_offsets); free(row_overlaps); free(empty_seqs);
    return out;
}

/* barb200_trace_ends' layout for every end; right_end_indexes == NULL: independent ends. Returns 0. */
int oracle_trace_ends(const oracle_params_t *p, int64_t end_no, const int64_t *end_lengths, char ***end_strings,
                      int **end_string_lengths, int64_t **right_end_indexes, int64_t **right_end_row_indexes, int64_t **overlaps,
                      int64_t window_size, int64_t max_prog_rows, double max_prog_length_diff, int64_t **trace_out, int64_t *n_words) {
    tbuf_t *bs = (tbuf_t *)calloc(end_no > 0 ? end_no : 1, sizeof(tbuf_t));
    wmsa_t *ws = (wmsa_t *)calloc(end_no > 0 ? end_no : 1, sizeof(wmsa_t));
    float **cs = (float **)malloc(sizeof(float *) * (end_no > 0 ? end_no : 1));
    for (int64_t i = 0; i < end_no; ++i) {
        oracle_msa_t *m = trace_end(p, end_strings[i], end_string_lengths[i], end_lengths[i], window_size, max_prog_rows,
                                    max_prog_length_diff, &bs[i]);
        ws[i].m = *m; ws[i].stride = m->column_no; free(m);
        cs[i] = column_scores(&ws[i]);
    }
    if (right_end_indexes)                                     /* :781-793 */
        for (int64_t i = 0; i < end_no; ++i)
            for (int64_t j = 0; j < ws[i].m.seq_no; ++j) {
                int64_t re = right_end_indexes[i][j], rr = right_end_row_indexes[i][j];
                if (re > i || (re == i && rr > j)) trim(j, &ws[i], cs[i], rr, &ws[re], cs[re], overlaps[i][j]);
            }
    for (int64_t i = 0; i < end_no; ++i) {
        const size_t nb = (size_t)ws[i].m.seq_no * ws[i].m.column_no, nwm = (nb + 7) / 8;
        tpush(&bs[i], ws[i].m.seq_no); tpush(&bs[i], ws[i].m.column_no);
        const size_t at = bs[i].n;
        for (size_t k = 0; k < nwm; ++k) tpush(&bs[i], 0);
        memcpy(bs[i].w + at, ws[i].m.msa, nb);
        trace_out[i] = bs[i].w; n_words[i] = (int64_t)bs[i].n;
        free(cs[i]); free(ws[i].m.seq_lens); free(ws[i].m.msa);
    }
    free(bs); free(ws); free(cs);
    return 0;
}
