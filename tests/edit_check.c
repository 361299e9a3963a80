/* Serial CPU statement of the edit metric of approximate positions, for large inputs.  Test infrastructure
 * only.  Deliberately a different route from the device's: no suffix array, no pieces and no band; per query
 * and document, one reversed Sellers column sweep (Sellers 1980) over the whole document with Ukkonen's cut-off.
 *
 * Column t holds C[r] = min over e of ED(q[m - r, m), T[t, e)) for r = 0..m, e <= the document's end, saturated
 * at k + 1; C[m] is dist(t).  Column end = the document's end: C[r] = r.  Column t from column t + 1 (P):
 * C[0] = 0, C[r] = min(P[r] + 1, C[r - 1] + 1, P[r - 1] + [q[m - r] != T[t]]).  Entries above the last one
 * <= k (lact) stay above k in the next column beyond lact + 1, so only r <= lact + 1 is computed. */
#include <stdint.h>
#include <stdlib.h>

/* Queries [q0, q1) cut at q_off; ndocs = 0: a single text.  counts[q - q0] = the occurrences of query q; when
 * pos is non-NULL, the occurrences of the queries in order by ascending p go to pos / dist (dist may be NULL).
 * Returns the sum of the counts, or UINT64_MAX when the column cannot be allocated. */
uint64_t edit_check(const uint8_t *text, uint64_t n, const uint32_t *starts, uint64_t ndocs,
                    const uint8_t *queries, const uint64_t *q_off, uint64_t q0, uint64_t q1, uint32_t k,
                    uint64_t *counts, uint32_t *pos, uint32_t *dist) {
    uint64_t total = 0;
    const uint64_t nd = ndocs ? ndocs : 1;
    for (uint64_t q = q0; q < q1; q++) {
        const uint8_t *pat = queries + q_off[q];
        const uint64_t m = q_off[q + 1] - q_off[q];
        const uint32_t inf = k + 1;
        uint32_t *col = malloc((m + 2) * sizeof *col);
        if (!col) return UINT64_MAX;
        uint64_t c = 0;
        for (uint64_t d = 0; d < nd && m > 0; d++) {
            const uint64_t s = ndocs ? starts[d] : 0, e = (ndocs && d + 1 < ndocs) ? starts[d + 1] : n;
            uint64_t lact = m < k ? m : k;                       /* column e: C[r] = r */
            for (uint64_t r = 0; r <= lact; r++) col[r] = (uint32_t)r;
            if (lact < m) col[lact + 1] = inf;
            /* hits of this document come out by descending p: written in place, reversed afterwards */
            const uint64_t first = total + c;
            for (uint64_t t = e; t-- > s;) {
                const uint8_t ch = text[t];
                const uint64_t top = lact + 1 <= m ? lact + 1 : m;
                uint32_t diag = col[0], left = 0;                /* P[r - 1]; C[r - 1] */
                col[0] = 0;
                for (uint64_t r = 1; r <= top; r++) {
                    const uint32_t prev = col[r];
                    uint32_t v = prev + 1;
                    if (left + 1 < v) v = left + 1;
                    const uint32_t sub = diag + (pat[m - r] != ch);
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
        counts[q - q0] = c;
        total += c;
    }
    return total;
}
