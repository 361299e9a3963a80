/* Serial CPU statement of the alignments of approximate hits (B200SA_APPROX_ALIGN), for large inputs.  Test
 * infrastructure only.  Deliberately a different route from the device's: no band and no shuffles; per hit one
 * row-major DP over every column t in [p, C], C = min(E, p + m + d + 1), with values saturated at d + 1, and the
 * canonical walk over the stored values.  Column E has D(x, E) = m - x; when C < E, column C holds d + 1 (any
 * path through it leaves the diagonals [-d, d], so it costs more than d).
 *
 * match(x, t): T[t] == Q[x], or with iupac the text byte in the class of the IUPAC code Q[x] (only uppercase
 * A C G T in the text).  Q is q, or rc(q) on a minus hit. */
#include <stdint.h>
#include <stdlib.h>

static uint32_t cls(uint8_t b) {                     /* an IUPAC code's class as a mask A 1, C 2, G 4, T 8 */
    switch (b | 0x20) {
    case 'a': return 1;
    case 'c': return 2;
    case 'g': return 4;
    case 't': case 'u': return 8;
    case 'r': return 5;
    case 'y': return 10;
    case 's': return 6;
    case 'w': return 9;
    case 'k': return 12;
    case 'm': return 3;
    case 'b': return 14;
    case 'd': return 13;
    case 'h': return 11;
    case 'v': return 7;
    case 'n': return 15;
    default: return 0;
    }
}

static uint8_t comp(uint8_t b, int iupac) {
    static const char *pairs = "ATTACGGCatta" "cggc";
    for (int i = 0; i < 16; i += 2)
        if (pairs[i] == b) return (uint8_t)pairs[i + 1];
    if (iupac) {
        static const char *more = "UARYYRKMMKBVVBDHHD" "uaryyrkmmkbvvbdhhd";
        for (int i = 0; i < 36; i += 2)
            if (more[i] == b) return (uint8_t)more[i + 1];
    }
    return b;
}

static int miss(uint8_t t, uint8_t q, int iupac) {
    if (!iupac) return t != q;
    const uint32_t bit = t == 'A' ? 1u : t == 'C' ? 2u : t == 'G' ? 4u : t == 'T' ? 8u : 0u;
    return (bit & cls(q)) == 0;
}

/* Hits h of query hq[h] at hp[h] with distance hd[h] (bit 31: minus).  ndocs = 0: a single text.  counts[h] =
 * the hit's operations; when words is non-NULL they go there in order (BAM words len << 4 | code, bit 31 on a
 * minus hit).  Returns the sum of the counts, or UINT64_MAX when the DP cannot be allocated or a walk's cost
 * differs from its hit's distance. */
uint64_t align_check(const uint8_t *text, uint64_t n, const uint32_t *starts, uint64_t ndocs, const uint8_t *queries,
                     const uint64_t *q_off, const uint32_t *hq, const uint32_t *hp, const uint32_t *hd, uint64_t nh,
                     int edit, int iupac, uint32_t *counts, uint32_t *words) {
    uint64_t total = 0;
    for (uint64_t h = 0; h < nh; h++) {
        const uint8_t *q = queries + q_off[hq[h]];
        const uint64_t m = q_off[hq[h] + 1] - q_off[hq[h]], p = hp[h];
        const int minus = hd[h] >> 31;
        const uint32_t d = hd[h] & 0x7FFFFFFFu, inf = d + 1;
        uint8_t *Q = malloc(m + 1);
        if (!Q) return UINT64_MAX;
        for (uint64_t x = 0; x < m; x++) Q[x] = minus ? comp(q[m - 1 - x], iupac) : q[x];
        uint64_t lo = 0, hi = ndocs;                   /* E: the end of p's document */
        while (hi - lo > 1) {
            const uint64_t mid = (lo + hi) / 2;
            if (starts[mid] <= p) lo = mid; else hi = mid;
        }
        const uint64_t E = (ndocs && lo + 1 < ndocs) ? starts[lo + 1] : n;
        uint32_t cnt = 0, code = 0, len = 0, cost = 0;
#define PUSH(c)                                                                              \
    do {                                                                                     \
        if ((c) == code) { len++; break; }                                                   \
        if (len) { if (words) words[total + cnt] = len << 4 | code | (minus ? 0x80000000u : 0u); cnt++; } \
        code = (c);                                                                          \
        len = 1;                                                                             \
    } while (0)
        if (!edit) {
            for (uint64_t x = 0; x < m; x++) {
                const int mm = miss(text[p + x], Q[x], iupac);
                cost += mm;
                PUSH(mm ? 8u : 7u);
            }
        } else {
            const uint64_t C = E < p + m + d + 1 ? E : p + m + d + 1, w = C - p + 1;
            uint32_t *D = malloc((m + 1) * w * sizeof *D);
            if (!D) { free(Q); return UINT64_MAX; }
#define AT(x, u) D[(x) * w + (u)]
            for (uint64_t u = 0; u < w; u++) AT(m, u) = (u + 1 < w || C == E) ? 0 : inf;
            for (uint64_t x = m; x-- > 0;) {
                AT(x, w - 1) = (C == E && m - x < inf) ? (uint32_t)(m - x) : inf;
                for (uint64_t u = w - 1; u-- > 0;) {
                    uint32_t v = AT(x + 1, u + 1) + (uint32_t)miss(text[p + u], Q[x], iupac);
                    if (AT(x + 1, u) + 1 < v) v = AT(x + 1, u) + 1;
                    if (AT(x, u + 1) + 1 < v) v = AT(x, u + 1) + 1;
                    AT(x, u) = v < inf ? v : inf;
                }
            }
            uint64_t x = 0, u = 0;
            if (AT(0, 0) != d) cost = ~0u;
            while (x < m && cost != ~0u) {
                const uint32_t v = AT(x, u);
                const int mm = p + u < E ? miss(text[p + u], Q[x], iupac) : 1;
                if (p + u < E && u + 1 < w && v == AT(x + 1, u + 1) + (uint32_t)mm) {
                    cost += mm;
                    PUSH(mm ? 8u : 7u);
                    x++;
                    u++;
                } else if (v == AT(x + 1, u) + 1) {
                    cost++;
                    PUSH(1u);
                    x++;
                } else {
                    cost++;
                    PUSH(2u);
                    u++;
                }
            }
#undef AT
            free(D);
        }
        if (len) { if (words) words[total + cnt] = len << 4 | code | (minus ? 0x80000000u : 0u); cnt++; }
#undef PUSH
        free(Q);
        if (cost != d) return UINT64_MAX;
        counts[h] = cnt;
        total += cnt;
    }
    return total;
}
