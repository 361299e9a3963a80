/* bwt_check.c -- the serial statement of the Burrows-Wheeler transform of documents (include/b200sa.h)
 * for large inputs: the forward transform from SA / G and doc_starts, and the inverse by the LF walk.
 * Test infrastructure only. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* document of p: the last d with starts[d] <= p */
static uint32_t doc_of(const uint32_t *starts, uint32_t k, uint32_t p) {
    uint32_t lo = 0, hi = k;
    while (hi - lo > 1) {
        uint32_t mid = lo + (hi - lo) / 2;
        if (starts[mid] <= p) lo = mid; else hi = mid;
    }
    return lo;
}

/* bwt (n bytes), term_rows (k); returns r, the runs of the full L of n + k symbols (256 + d for $_d). */
int64_t bwt_forward(uint64_t n, const uint8_t *text, const uint32_t *g, const uint32_t *starts, uint32_t k,
                    uint8_t *bwt, uint32_t *term_rows) {
    uint64_t u = 0, runs = 0;
    uint32_t prev = 0xffffffffu;
    for (uint64_t i = 0; i < n + k; i++) {
        uint32_t s;
        if (i < k) {
            uint64_t e = i + 1 < k ? starts[i + 1] : n;
            s = e > starts[i] ? text[e - 1] : 256u + (uint32_t)i;
        } else {
            uint32_t p = g[i - k], d = doc_of(starts, k, p);
            s = p == starts[d] ? 256u + d : text[p - 1];
        }
        if (s >= 256u) term_rows[s - 256u] = (uint32_t)i;
        else bwt[u++] = (uint8_t)s;
        runs += s != prev;
        prev = s;
    }
    return (int64_t)runs;
}

/* The documents of (bwt, term_rows) by the LF walk: LF(row) = d for L = $_d, else k + C[c] + the number of
 * c before row.  Walking LF from row d reads D_d backwards.  Writes text (n bytes) and starts (k); returns
 * 0, or 1 when the input is not the transform of any documents. */
int bwt_inverse(uint64_t n, uint32_t k, const uint8_t *bwt, const uint32_t *term_rows, uint8_t *text,
                uint32_t *starts) {
    uint64_t rows = n + k;
    int32_t *termof = malloc(rows * sizeof *termof);
    uint32_t *lf = malloc(rows * sizeof *lf);
    uint8_t *lb = malloc(rows ? rows : 1);
    uint64_t *len = calloc(k ? k : 1, sizeof *len);
    int bad = !termof || !lf || !lb || !len;
    if (!bad) {
        for (uint64_t i = 0; i < rows; i++) termof[i] = -1;
        for (uint32_t d = 0; d < k && !bad; d++) {
            if (term_rows[d] >= rows || termof[term_rows[d]] >= 0) bad = 1;
            else termof[term_rows[d]] = (int32_t)d;
        }
    }
    if (!bad) {
        uint64_t cnt[257] = {0}, occ[256] = {0};
        for (uint64_t u = 0; u < n; u++) cnt[bwt[u] + 1]++;
        for (int c = 0; c < 256; c++) cnt[c + 1] += cnt[c];
        uint64_t u = 0;
        for (uint64_t i = 0; i < rows; i++) {
            if (termof[i] >= 0) {
                lf[i] = (uint32_t)termof[i];
            } else {
                uint8_t c = bwt[u++];
                lb[i] = c;
                lf[i] = (uint32_t)(k + cnt[c] + occ[c]++);
            }
        }
        /* lengths: from row d, LF until the row whose L is $_d; no other terminator on the way */
        uint64_t seen = 0;
        for (uint32_t d = 0; d < k && !bad; d++) {
            uint64_t x = d, l = 0;
            while (termof[x] < 0 && l <= rows) { x = lf[x]; l++; }
            if (termof[x] != (int32_t)d) bad = 1;
            len[d] = l;
            seen += l + 1;
        }
        if (!bad && seen != rows) bad = 1;
        if (!bad) {
            uint64_t at = 0;
            for (uint32_t d = 0; d < k; d++) {
                starts[d] = (uint32_t)at;
                uint64_t x = d, w = at + len[d];
                for (uint64_t j = 0; j < len[d]; j++) {
                    text[--w] = lb[x];
                    x = lf[x];
                }
                at += len[d];
            }
        }
    }
    free(termof);
    free(lf);
    free(lb);
    free(len);
    return bad;
}
