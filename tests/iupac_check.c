/* Serial CPU statement of IUPAC queries in approximate positions (B200SA_APPROX_IUPAC), for large inputs.  Test
 * infrastructure only.  Deliberately a different route from the device's: no suffix array and no pieces.  Per
 * query and document, the Hamming metric counts class mismatches over every window, and the edit metric runs one
 * reversed Sellers column sweep (Sellers 1980) over the whole document with Ukkonen's cut-off.
 *
 * A symbol's class is a mask of bases (A 1, C 2, G 4, T 8); a text byte is in it iff it is an uppercase A C G T
 * whose bit is set.  A query byte that is no IUPAC code has the empty class.  Edit columns as in edit_check.c:
 * column t holds C[r] = min over e of ED(q[m - r, m), T[t, e)), e <= the document's end, saturated at k + 1. */
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

/* Queries [q0, q1) cut at q_off; ndocs = 0: a single text; edit = 0: mis(p), else dist(p).  counts[q - q0] = the
 * occurrences of query q; when pos is non-NULL, the occurrences of the queries in order by ascending p go to
 * pos / dist (dist may be NULL).  Returns the sum of the counts, or UINT64_MAX when memory runs out. */
uint64_t iupac_check(const uint8_t *text, uint64_t n, const uint32_t *starts, uint64_t ndocs, const uint8_t *queries,
                     const uint64_t *q_off, uint64_t q0, uint64_t q1, uint32_t k, int edit, uint64_t *counts,
                     uint32_t *pos, uint32_t *dist) {
    uint64_t total = 0;
    const uint64_t nd = ndocs ? ndocs : 1;
    for (uint64_t q = q0; q < q1; q++) {
        const uint8_t *pat = queries + q_off[q];
        const uint64_t m = q_off[q + 1] - q_off[q];
        const uint32_t inf = k + 1;
        uint32_t *col = malloc((m + 2) * sizeof *col);
        unsigned *cls = malloc((m + 1) * sizeof *cls);
        if (!col || !cls) {
            free(col);
            free(cls);
            return UINT64_MAX;
        }
        for (uint64_t x = 0; x < m; x++) cls[x] = query_class(pat[x]);
        uint64_t c = 0;
        for (uint64_t d = 0; d < nd && m > 0; d++) {
            const uint64_t s = ndocs ? starts[d] : 0, e = (ndocs && d + 1 < ndocs) ? starts[d + 1] : n;
            if (!edit) {
                for (uint64_t p = s; p + m <= e; p++) {
                    uint32_t mis = 0;
                    for (uint64_t x = 0; x < m && mis <= k; x++) mis += !(text_bit(text[p + x]) & cls[x]);
                    if (mis <= k) {
                        if (pos) {
                            pos[total + c] = (uint32_t)p;
                            if (dist) dist[total + c] = mis;
                        }
                        c++;
                    }
                }
                continue;
            }
            uint64_t lact = m < k ? m : k;                       /* column e: C[r] = r */
            for (uint64_t r = 0; r <= lact; r++) col[r] = (uint32_t)r;
            if (lact < m) col[lact + 1] = inf;
            const uint64_t first = total + c;                    /* hits come by descending p; reversed below */
            for (uint64_t t = e; t-- > s;) {
                const unsigned bit = text_bit(text[t]);
                const uint64_t top = lact + 1 <= m ? lact + 1 : m;
                uint32_t diag = col[0], left = 0;                /* P[r - 1]; C[r - 1] */
                col[0] = 0;
                for (uint64_t r = 1; r <= top; r++) {
                    const uint32_t prev = col[r];
                    uint32_t v = prev + 1;
                    if (left + 1 < v) v = left + 1;
                    const uint32_t sub = diag + !(bit & cls[m - r]);
                    if (sub < v) v = sub;
                    if (v > inf) v = inf;
                    col[r] = v;
                    diag = prev;
                    left = v;
                }
                lact = top;
                while (lact > 0 && col[lact] > k) lact--;
                if (lact < m) col[lact + 1] = inf;
                if (lact == m) {
                    if (pos) {
                        pos[total + c] = (uint32_t)t;
                        if (dist) dist[total + c] = col[m];
                    }
                    c++;
                }
            }
            if (pos)
                for (uint64_t a = first, b = total + c; a + 1 < b; a++, b--) {
                    uint32_t x = pos[a];
                    pos[a] = pos[b - 1];
                    pos[b - 1] = x;
                    if (dist) {
                        x = dist[a];
                        dist[a] = dist[b - 1];
                        dist[b - 1] = x;
                    }
                }
        }
        free(col);
        free(cls);
        counts[q - q0] = c;
        total += c;
    }
    return total;
}
