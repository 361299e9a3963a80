/* Serial CPU statement of the longest previous factor and the LZ77 factorization of a table
 * (include/b200sa.h, DESIGN.md 6b f-12) for inputs too large for the Python model, and a decoder that
 * rebuilds the text from the factors.  It shares no route with the device code: psv / nsv and their LCPs
 * come from one stack sweep in each direction (the LCP to the stack's top carried as the stack shrinks),
 * the parse is the serial walk.  Test infrastructure only. */
#include <stdint.h>
#include <stdlib.h>

#define LZ_LITERAL 0xFFFFFFFFu

/* lpf / src in text order; the factors, of which the first `cap` are written where the arrays are given.
 * Returns z, or -1 when out of memory. */
int64_t lz_check(uint64_t n, const uint32_t *sa, const uint32_t *lcp, uint32_t *lpf, uint32_t *src,
                 uint32_t *start, uint32_t *len, uint32_t *fsrc, uint64_t cap) {
    uint32_t *st = malloc((n + 1) * sizeof *st), *lk = malloc((n + 1) * sizeof *lk);
    uint32_t *lL = malloc((n + 1) * sizeof *lL), *pv = malloc((n + 1) * sizeof *pv);
    if (!st || !lk || !lL || !pv) { free(st); free(lk); free(lL); free(pv); return -1; }
    /* left to right: the stack holds ranks of increasing position, lk[i] = lcp(st[i], st[i+1]) and, for
     * the top, lcp(top, r) once r is reached */
    uint64_t k = 0;
    for (uint64_t r = 0; r < n; r++) {
        uint32_t cur = r ? lcp[r] : 0;
        while (k && sa[st[k - 1]] > sa[r]) {
            k--;
            if (k && lk[k - 1] < cur) cur = lk[k - 1];
        }
        pv[r] = k ? sa[st[k - 1]] : LZ_LITERAL;
        lL[r] = k ? cur : 0;
        if (k) lk[k - 1] = cur;
        st[k++] = (uint32_t)r;
    }
    /* right to left, the same with lcp(r, r + 1) */
    k = 0;
    for (uint64_t i = n; i-- > 0;) {
        uint32_t cur = i + 1 < n ? lcp[i + 1] : 0;
        while (k && sa[st[k - 1]] > sa[i]) {
            k--;
            if (k && lk[k - 1] < cur) cur = lk[k - 1];
        }
        const uint32_t lR = k ? cur : 0, p = sa[i];
        lpf[p] = lL[i] > lR ? lL[i] : lR;
        if (lL[i] >= lR && lL[i] > 0) src[p] = pv[i];
        else src[p] = lR > 0 ? sa[st[k - 1]] : LZ_LITERAL;
        if (k) lk[k - 1] = cur;
        st[k++] = (uint32_t)i;
    }
    free(st); free(lk); free(lL); free(pv);
    int64_t z = 0;
    for (uint64_t p = 0; p < n; z++) {
        const uint32_t l = lpf[p] > 1 ? lpf[p] : 1;
        if ((uint64_t)z < cap) {
            if (start) start[z] = (uint32_t)p;
            if (len) len[z] = l;
            if (fsrc) fsrc[z] = src[p];
        }
        p += l;
    }
    return z;
}

/* Rebuilds n bytes into out from the z factors; a literal takes the next byte of `literals`.  Returns 0,
 * or the 1-based index of the first factor that is malformed (not contiguous, a source at or after its
 * start, a literal longer than 1, past the end). */
int64_t lz_decode(uint64_t n, uint64_t z, const uint32_t *start, const uint32_t *len, const uint32_t *src,
                  const uint8_t *literals, uint8_t *out) {
    uint64_t pos = 0, lit = 0;
    for (uint64_t i = 0; i < z; i++) {
        const uint64_t s = start[i], l = len[i];
        if (s != pos || l == 0 || s + l > n) return (int64_t)i + 1;
        if (src[i] == LZ_LITERAL) {
            if (l != 1) return (int64_t)i + 1;
            out[s] = literals[lit++];
        } else {
            if (src[i] >= s) return (int64_t)i + 1;
            for (uint64_t j = 0; j < l; j++) out[s + j] = out[src[i] + j];
        }
        pos = s + l;
    }
    return pos == n ? 0 : (int64_t)z + 1;
}
