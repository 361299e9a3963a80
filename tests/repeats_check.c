/* Serial CPU statement of the repeats of a table (include/b200sa.h, DESIGN.md 6b f-11) for inputs too
 * large for the Python model.  It shares no route with the device code: the runs are walked rank by
 * rank with a running min / max, the spans are swept off a byte mask.  Test infrastructure only. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static uint32_t lam(const uint32_t *lcp, uint64_t n, uint64_t i) { return i < n ? lcp[i] : 0; }

/* document of p: the last d with starts[d] <= p */
static uint32_t doc_of(const uint32_t *starts, uint32_t ndocs, uint32_t p) {
    uint32_t lo = 0, hi = ndocs;
    while (hi - lo > 1) {
        uint32_t mid = lo + (hi - lo) / 2;
        if (starts[mid] <= p) lo = mid; else hi = mid;
    }
    return lo;
}

/* The runs at L: returns their number; writes the first `cap` of them where the arrays are given. */
uint64_t repeats_check_runs(uint64_t n, const uint32_t *sa, const uint32_t *lcp, uint32_t L, uint32_t *start,
                            uint32_t *end, uint32_t *first, uint32_t *last, uint64_t cap) {
    uint64_t k = 0, a = 0;
    while (a < n) {
        uint64_t b = a + 1;
        uint32_t lo = sa[a], hi = sa[a];
        while (b < n && lcp[b] >= L) {
            if (sa[b] < lo) lo = sa[b];
            if (sa[b] > hi) hi = sa[b];
            b++;
        }
        if (b - a >= 2) {
            if (k < cap) {
                if (start) start[k] = (uint32_t)a;
                if (end) end[k] = (uint32_t)b;
                if (first) first[k] = lo;
                if (last) last[k] = hi;
            }
            k++;
        }
        a = b;
    }
    return k;
}

/* The spans of `mode` (0 any, 1 earlier, 2 other document, 3 earlier document; starts = NULL: a single
 * text).  Returns their number, writes the first `cap` and *covered.  -1: out of memory. */
int64_t repeats_check_spans(uint64_t n, const uint32_t *sa, const uint32_t *lcp, const uint32_t *starts,
                            uint32_t ndocs, uint32_t L, int mode, uint32_t *begin, uint32_t *end, uint64_t cap,
                            uint64_t *covered) {
    uint8_t *mask = calloc(n + 1, 1), *cut = calloc(n + 2, 1);
    if (!mask || !cut) { free(mask); free(cut); return -1; }
    for (uint32_t d = 0; starts && d < ndocs; d++) cut[starts[d]] = 1;
    cut[0] = cut[n] = 1;
    uint64_t a = 0;
    while (a < n) {
        uint64_t b = a + 1;
        uint32_t lo = sa[a], hi = sa[a];
        while (b < n && lam(lcp, n, b) >= L) {
            if (sa[b] < lo) lo = sa[b];
            if (sa[b] > hi) hi = sa[b];
            b++;
        }
        for (uint64_t r = a; b - a >= 2 && r < b; r++) {
            const uint32_t p = sa[r];
            int f = 1;
            if (mode == 1) f = p != lo;
            if (mode >= 2) {
                const uint32_t d = doc_of(starts, ndocs, p), ds = starts[d];
                const uint64_t de = d + 1 < ndocs ? starts[d + 1] : n;
                f = lo < ds || (mode == 2 && hi >= de);
            }
            if (f) memset(mask + p, 1, L);                 /* p + L <= n: the gram lies inside p's document */
        }
        a = b;
    }
    uint64_t k = 0, cov = 0;
    for (uint64_t x = 0; x < n; x++) {
        if (!mask[x]) continue;
        cov++;
        if (x == 0 || !mask[x - 1] || cut[x]) {
            if (k < cap && begin) begin[k] = (uint32_t)x;
        }
        if (x + 1 == n || !mask[x + 1] || cut[x + 1]) {
            if (k < cap && end) end[k] = (uint32_t)x + 1;
            k++;
        }
    }
    *covered = cov;
    free(mask);
    free(cut);
    return (int64_t)k;
}
