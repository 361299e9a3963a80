/* Serial CPU statement of matching statistics over a (generalized) suffix array, for large inputs.  Test
 * infrastructure only.  Deliberately a different route from the device's: per pattern position, a plain
 * binary search for the insertion point with whole compares from byte 0, the longest match as the better
 * of the two neighbours, and the range by two more binary searches on the matched string (no LCP array). */
#include <stdint.h>
#include <string.h>

typedef struct {
    const uint8_t *text;
    uint64_t n;
    const uint32_t *starts;
    uint64_t ndocs;
    const uint32_t *sa;
} idx_t;

static uint64_t suffix_end(const idx_t *x, uint32_t p) {
    uint64_t lo = 0, hi = x->ndocs;              /* last d with starts[d] <= p */
    if (x->ndocs == 0) return x->n;
    while (hi - lo > 1) {
        uint64_t mid = lo + (hi - lo) / 2;
        if (x->starts[mid] <= p) lo = mid; else hi = mid;
    }
    return lo + 1 < x->ndocs ? x->starts[lo + 1] : x->n;
}

/* common prefix of q[0, m) and the suffix at rank r; *cmp < 0, 0, > 0 as q compares to the suffix
 * truncated to m bytes (0: the suffix starts with q) */
static uint64_t common(const idx_t *x, uint64_t r, const uint8_t *q, uint64_t m, int *cmp) {
    uint32_t p = x->sa[r];
    uint64_t ls = suffix_end(x, p) - p, l = ls < m ? ls : m, k = 0;
    const uint8_t *s = x->text + p;
    while (k < l && q[k] == s[k]) k++;
    if (k == m) *cmp = 0;
    else if (k == ls) *cmp = 1;
    else *cmp = q[k] < s[k] ? -1 : 1;
    return k;
}

/* first rank whose suffix, truncated to m bytes, is >= q (upper = 0) or > q (upper = 1) */
static uint64_t bound(const idx_t *x, const uint8_t *q, uint64_t m, int upper) {
    uint64_t lo = 0, hi = x->n;
    while (lo < hi) {
        uint64_t mid = lo + (hi - lo) / 2;
        int c;
        common(x, mid, q, m, &c);
        if (upper ? c >= 0 : c > 0) lo = mid + 1; else hi = mid;
    }
    return lo;
}

/* len / start / end (start and end may be NULL) of pattern positions [x0, x1) of the queries cut at q_off.
 * ndocs = 0: a single text. */
void match_check(const uint8_t *text, uint64_t n, const uint32_t *starts, uint64_t ndocs, const uint32_t *sa,
                 const uint8_t *queries, const uint64_t *q_off, uint64_t nq, uint64_t x0, uint64_t x1,
                 uint32_t *len, uint32_t *start, uint32_t *end) {
    idx_t ix = {text, n, starts, ndocs, sa};
    uint64_t q = 0;
    for (uint64_t x = x0; x < x1; x++) {
        while (q + 1 < nq && q_off[q + 1] <= x) q++;
        const uint8_t *pat = queries + x;
        uint64_t m = q_off[q + 1] - x, best = 0;
        uint64_t ins = n ? bound(&ix, pat, m, 0) : 0;
        int c;
        if (ins < n) best = common(&ix, ins, pat, m, &c);
        if (ins > 0) {
            uint64_t b = common(&ix, ins - 1, pat, m, &c);
            if (b > best) best = b;
        }
        len[x - x0] = (uint32_t)best;
        if (start) {
            start[x - x0] = best ? (uint32_t)bound(&ix, pat, best, 0) : 0;
            end[x - x0] = best ? (uint32_t)bound(&ix, pat, best, 1) : 0;
        }
    }
}
