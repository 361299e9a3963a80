/* docs_check.c -- CPU checker of a separator-free generalized suffix array (b200sa_docs_build)
 * for inputs too large for the Python brute force.  Test infrastructure only.
 *
 * docs_check(text, n, starts, ndocs, g, glcp) verifies by direct compare that
 *   - g is a permutation of 0..n-1;
 *   - every adjacent pair is strictly in (document suffix, document) order;
 *   - glcp[0] = 0 and glcp[i] is the common prefix length of the document suffixes g[i-1], g[i].
 * Returns 0 if all hold, else a negative code: -1 - i for the first bad rank i of the order or
 * glcp check, or INT64_MIN for a non-permutation.  glcp may be NULL. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static uint64_t doc_of(const uint32_t *starts, uint64_t ndocs, uint64_t p) {
    uint64_t lo = 0, hi = ndocs;                  /* last d with starts[d] <= p */
    while (hi - lo > 1) {
        uint64_t mid = lo + (hi - lo) / 2;
        if (starts[mid] <= p) lo = mid; else hi = mid;
    }
    return lo;
}

int64_t docs_check(const uint8_t *text, uint64_t n, const uint32_t *starts, uint64_t ndocs, const uint32_t *g,
                   const uint32_t *glcp) {
    uint8_t *seen = calloc(n ? n : 1, 1);
    if (!seen) return INT64_MIN;
    for (uint64_t i = 0; i < n; i++) {
        if (g[i] >= n || seen[g[i]]) { free(seen); return INT64_MIN; }
        seen[g[i]] = 1;
    }
    free(seen);
    if (n > 0 && glcp && glcp[0] != 0) return -1;
    for (uint64_t i = 1; i < n; i++) {
        uint64_t a = g[i - 1], b = g[i];
        uint64_t da = doc_of(starts, ndocs, a), db = doc_of(starts, ndocs, b);
        uint64_t ra = (da + 1 < ndocs ? starts[da + 1] : n) - a, rb = (db + 1 < ndocs ? starts[db + 1] : n) - b;
        uint64_t m = ra < rb ? ra : rb, l = 0;
        while (l < m && text[a + l] == text[b + l]) l++;
        int ordered = l < m ? text[a + l] < text[b + l] : (ra < rb || (ra == rb && da < db));
        if (!ordered || (glcp && glcp[i] != l)) return -1 - (int64_t)i;
    }
    return 0;
}
