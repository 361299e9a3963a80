/* Serial CPU statement of fixed symbols in IUPAC queries (B200SA_APPROX_FIXED), for large inputs.  Test
 * infrastructure only.  Deliberately a different route from the device's: no suffix array and no pieces.  Per
 * query and document, the Hamming metric tests every window, and the edit metric runs one reversed Sellers column
 * sweep over the whole document, every column in full (the constraints break the monotonicity a cut-off needs).
 *
 * Classes as in iupac_check.c; a query byte is fixed iff it is a lowercase letter.  Column t holds
 * C[r] = D(x, t) for x = m - r: the least cost of aligning q[x, m) to a T[t, e), e <= the document's end, under the
 * rules -- a fixed q[x] takes no X and no I, and no D at (x, t) when q[x] or q[x - 1] is fixed -- saturated at
 * k + 1 (also where no alignment keeps them). */
#include <stdint.h>
#include <stdlib.h>

static unsigned text_bit(uint8_t t) {
    return t == 'A' ? 1u : t == 'C' ? 2u : t == 'G' ? 4u : t == 'T' ? 8u : 0u;
}

static unsigned query_class(uint8_t b) {
    switch (b >= 'a' && b <= 'z' ? b - 32 : b) {
    case 'A': return 1;
    case 'C': return 2;
    case 'G': return 4;
    case 'T': case 'U': return 8;
    case 'R': return 5;
    case 'Y': return 10;
    case 'S': return 6;
    case 'W': return 9;
    case 'K': return 12;
    case 'M': return 3;
    case 'B': return 14;
    case 'D': return 13;
    case 'H': return 11;
    case 'V': return 7;
    case 'N': return 15;
    default: return 0;
    }
}

static uint32_t min2(uint32_t a, uint32_t b) { return a < b ? a : b; }

/* Queries [q0, q1) cut at q_off; ndocs = 0: a single text; edit = 0: mis(p) over the free symbols, else dist(p).
 * counts[q - q0] = the occurrences of query q; when pos is non-NULL, the occurrences of the queries in order by
 * ascending p go to pos / dist (dist may be NULL).  Returns the sum of the counts, or UINT64_MAX when memory runs
 * out. */
uint64_t fixed_check(const uint8_t *text, uint64_t n, const uint32_t *starts, uint64_t ndocs, const uint8_t *queries,
                     const uint64_t *q_off, uint64_t q0, uint64_t q1, uint32_t k, int edit, uint64_t *counts,
                     uint32_t *pos, uint32_t *dist) {
    uint64_t total = 0;
    const uint64_t nd = ndocs ? ndocs : 1;
    for (uint64_t q = q0; q < q1; q++) {
        const uint8_t *pat = queries + q_off[q];
        const uint64_t m = q_off[q + 1] - q_off[q];
        const uint32_t inf = k + 1;
        uint32_t *col = malloc((m + 1) * sizeof *col);
        unsigned *cls = malloc((m + 1) * sizeof *cls);
        uint8_t *fx = malloc(m + 1);
        if (!col || !cls || !fx) {
            free(col);
            free(cls);
            free(fx);
            return UINT64_MAX;
        }
        for (uint64_t x = 0; x < m; x++) {
            cls[x] = query_class(pat[x]);
            fx[x] = pat[x] >= 'a' && pat[x] <= 'z';
        }
        uint64_t c = 0;
        for (uint64_t d = 0; d < nd && m > 0; d++) {
            const uint64_t s = ndocs ? starts[d] : 0, e = (ndocs && d + 1 < ndocs) ? starts[d + 1] : n;
            if (!edit) {
                for (uint64_t p = s; p + m <= e; p++) {
                    uint32_t mis = 0;
                    int ok = 1;
                    for (uint64_t x = 0; x < m && ok && mis <= k; x++) {
                        const int miss = !(text_bit(text[p + x]) & cls[x]);
                        if (miss && fx[x]) ok = 0;
                        mis += miss;
                    }
                    if (ok && mis <= k) {
                        if (pos) {
                            pos[total + c] = (uint32_t)p;
                            if (dist) dist[total + c] = mis;
                        }
                        c++;
                    }
                }
                continue;
            }
            col[0] = 0;                                          /* column e: only I moves */
            for (uint64_t r = 1; r <= m; r++) col[r] = fx[m - r] ? inf : min2(col[r - 1] + 1, inf);
            const uint64_t first = total + c;                    /* hits come by descending p; reversed below */
            for (uint64_t t = e; t-- > s;) {
                const unsigned bit = text_bit(text[t]);
                uint32_t diag = col[0];                          /* C_{t+1}[r - 1] */
                col[0] = 0;
                for (uint64_t r = 1; r <= m; r++) {
                    const uint64_t x = m - r;
                    const uint32_t prev = col[r];                /* C_{t+1}[r] */
                    const int miss = !(bit & cls[x]);
                    uint32_t v = inf;
                    if (!(fx[x] || (x > 0 && fx[x - 1]))) v = min2(v, prev + 1);      /* D */
                    if (!fx[x]) v = min2(v, col[r - 1] + 1);                          /* I */
                    if (!(fx[x] && miss)) v = min2(v, diag + (uint32_t)miss);          /* = or X */
                    col[r] = min2(v, inf);
                    diag = prev;
                }
                if (col[m] <= k) {
                    if (pos) {
                        pos[total + c] = (uint32_t)t;
                        if (dist) dist[total + c] = col[m];
                    }
                    c++;
                }
            }
            if (pos)
                for (uint64_t a = first, b = total + c; a + 1 < b; a++, b--) {
                    uint32_t y = pos[a];
                    pos[a] = pos[b - 1];
                    pos[b - 1] = y;
                    if (dist) {
                        y = dist[a];
                        dist[a] = dist[b - 1];
                        dist[b - 1] = y;
                    }
                }
        }
        free(col);
        free(cls);
        free(fx);
        counts[q - q0] = c;
        total += c;
    }
    return total;
}
