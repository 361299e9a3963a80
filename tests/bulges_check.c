/* The serial CPU statement of separate budgets for substitutions, DNA bulges and RNA bulges
 * (include/b200sa.h, B200SA_APPROX_BULGES), for large inputs.  Test infrastructure only.
 *
 * For every start p of every document and every query, a forward DP over the prefixes of the query:
 * H[x][u][i][e] is the least #X of an alignment of Q[0, x) to T[p, p + u) with at most i I (query bytes with no
 * text byte) and at most e D (text bytes with no query byte) moves.  p is an occurrence when some x = m cell with
 * p + u <= E (E the document's end) has H[m][u][r][d] <= t; dist(p) is the least H + i + e over those cells and
 * layers within t.  With iupac the query bytes are IUPAC codes matched against uppercase A C G T; with fixed the
 * lowercase symbols take no X or I and no D sits next to one.  A row whose every cell exceeds t ends the start. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static unsigned code_mask(unsigned b) {
    switch (b | 0x20u) {
    case 'a': return 1; case 'c': return 2; case 'g': return 4; case 't': case 'u': return 8;
    case 'r': return 5; case 'y': return 10; case 's': return 6; case 'w': return 9; case 'k': return 12;
    case 'm': return 3; case 'b': return 14; case 'd': return 13; case 'h': return 11; case 'v': return 7;
    case 'n': return 15; default: return 0;
    }
}

static int miss(unsigned t, unsigned q, int iupac) {
    if (!iupac) return t != q;
    unsigned bit = t == 'A' ? 1u : t == 'C' ? 2u : t == 'G' ? 4u : t == 'T' ? 8u : 0u;
    return (bit & code_mask(q)) == 0;
}

#define BIGV 1000000

/* Query q0 .. q1 - 1 of the blob; cnt[q - q0] gets each count; pos / dist (when non-NULL) the hits in (q, p)
 * order.  Returns the total, or ~0 when out of memory. */
uint64_t bulges_check(const uint8_t *text, uint64_t n, const uint32_t *starts, uint64_t ndocs, const uint8_t *blob,
                      const uint64_t *q_off, uint64_t q0, uint64_t q1, uint32_t t, uint32_t d, uint32_t r, int iupac,
                      int fixed, uint64_t *cnt, uint32_t *pos, uint32_t *dist) {
    uint64_t total = 0, mmax = 0;
    for (uint64_t q = q0; q < q1; q++)
        if (q_off[q + 1] - q_off[q] > mmax) mmax = q_off[q + 1] - q_off[q];
    const uint32_t NL = (r + 1) * (d + 1), W = d + r + 1;     /* cell b = u - x + r */
    int *H = malloc(sizeof(int) * (mmax + 1) * W * NL);
    uint8_t *fx = malloc(mmax + 1);
    if (!H || !fx) { free(H); free(fx); return ~0ull; }
    const uint64_t nd = ndocs ? ndocs : 1;
    for (uint64_t q = q0; q < q1; q++) {
        const uint8_t *Q = blob + q_off[q];
        const uint64_t m = q_off[q + 1] - q_off[q];
        uint64_t c = 0;
        for (uint64_t x = 0; x < m; x++) fx[x] = fixed && Q[x] >= 'a' && Q[x] <= 'z';
        for (uint64_t di = 0; di < nd && m > 0; di++) {
            const uint64_t s = ndocs ? starts[di] : 0, E = ndocs ? (di + 1 < ndocs ? starts[di + 1] : n) : n;
            for (uint64_t p = s; p < E; p++) {
                int alive = 1;
                for (uint64_t x = 0; x <= m && alive; x++) {
                    int low = BIGV;
                    for (uint32_t b = 0; b < W; b++) {
                        const int64_t u = (int64_t)x + b - r;
                        for (uint32_t i = 0; i <= r; i++)
                            for (uint32_t e = 0; e <= d; e++) {
                                int y = BIGV;
                                if (u >= 0 && p + (uint64_t)u <= E) {
                                    if (x == 0 && u == 0) y = 0;
                                    if (x > 0 && u > 0) {                       /* diagonal from (x-1, u-1), cell b */
                                        const int mi = miss(text[p + u - 1], Q[x - 1], iupac);
                                        if (!(fx[x - 1] && mi)) {
                                            const int h = H[((x - 1) * W + b) * NL + i * (d + 1) + e];
                                            if (h + mi < y) y = h + mi;
                                        }
                                    }
                                    if (x > 0 && i > 0 && !fx[x - 1] && b + 1 < W) {   /* I from (x-1, u), cell b+1 */
                                        const int h = H[((x - 1) * W + b + 1) * NL + (i - 1) * (d + 1) + e];
                                        if (h < y) y = h;
                                    }
                                    /* D from (x, u-1), cell b-1: not at x = m, nor next to a fixed symbol */
                                    if (e > 0 && b > 0 && u > 0 && x < m && !fx[x] && !(x > 0 && fx[x - 1])) {
                                        const int h = H[(x * W + b - 1) * NL + i * (d + 1) + e - 1];
                                        if (h < y) y = h;
                                    }
                                }
                                H[(x * W + b) * NL + i * (d + 1) + e] = y;
                                if (y < low) low = y;
                            }
                    }
                    if (low > (int)t) alive = 0;
                }
                if (!alive) continue;
                int best = BIGV;
                for (uint32_t b = 0; b < W; b++)
                    for (uint32_t i = 0; i <= r; i++)
                        for (uint32_t e = 0; e <= d; e++) {
                            const int h = H[(m * W + b) * NL + i * (d + 1) + e];
                            if (h <= (int)t && h + (int)(i + e) < best) best = h + (int)(i + e);
                        }
                if (best == BIGV) continue;
                if (pos) { pos[total] = (uint32_t)p; dist[total] = (uint32_t)best; }
                total++;
                c++;
            }
        }
        cnt[q - q0] = c;
    }
    free(H);
    free(fx);
    return total;
}
