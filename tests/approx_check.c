/* Serial CPU statement of approximate positions, for large inputs.  Test infrastructure only.  Deliberately a
 * different route from the device's: no suffix array and no pieces; per query, a sliding window over every
 * document with a Hamming count that stops above k. */
#include <stdint.h>

/* Queries [q0, q1) cut at q_off; ndocs = 0: a single text.  counts[q - q0] = the occurrences of query q; when
 * pos is non-NULL, the occurrences of the queries in order by ascending p go to pos / mis (mis may be NULL).
 * Returns the sum of the counts. */
uint64_t approx_check(const uint8_t *text, uint64_t n, const uint32_t *starts, uint64_t ndocs,
                      const uint8_t *queries, const uint64_t *q_off, uint64_t q0, uint64_t q1, uint32_t k,
                      uint64_t *counts, uint32_t *pos, uint32_t *mis) {
    uint64_t total = 0;
    const uint64_t nd = ndocs ? ndocs : 1;
    for (uint64_t q = q0; q < q1; q++) {
        const uint8_t *pat = queries + q_off[q];
        const uint64_t m = q_off[q + 1] - q_off[q];
        uint64_t c = 0;
        for (uint64_t d = 0; d < nd && m > 0; d++) {
            const uint64_t s = ndocs ? starts[d] : 0, e = (ndocs && d + 1 < ndocs) ? starts[d + 1] : n;
            for (uint64_t p = s; p + m <= e; p++) {
                uint32_t x = 0;
                for (uint64_t i = 0; i < m && x <= k; i++) x += text[p + i] != pat[i];
                if (x > k) continue;
                if (pos) {
                    pos[total + c] = (uint32_t)p;
                    if (mis) mis[total + c] = x;
                }
                c++;
            }
        }
        counts[q - q0] = c;
        total += c;
    }
    return total;
}
