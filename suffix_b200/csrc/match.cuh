// match.cuh -- matching statistics and super-maximal exact matches of query batches (DESIGN 6b f-10).
//
// For every pattern position x (a byte of the concatenated queries, inside query q with end E):
//   len[x]            the longest prefix of queries[x, E) that is a prefix of some suffix of the table
//   [start[x], end[x])  the range of the table whose suffixes start with that prefix (0, 0 when len = 0)
// One binary search per position gives both.  Invariant: the suffixes at ranks <= lo are < pattern and
// share llo bytes with it at lo; the suffixes at ranks >= hi are >= pattern and share lhi bytes at hi
// (lo = -1 and hi = n are virtual, sharing 0).  The table is sorted, so every suffix strictly between
// the bounds shares at least min(llo, lhi) bytes with the pattern and a probe starts comparing there.
// When the bounds meet, the two neighbours of the insertion point are the bounds themselves and the
// longest match is max(llo, lhi), at the bound that attains it (the witness w).  The range of the match
// is the LCP interval of depth len around w: the nearest lcp < len at or before w, and after w.
#pragma once
#include "docs.cuh"

namespace b200sa {

// bits of the q_off check word (reported through last_error)
constexpr uint32_t MATCH_BAD_FIRST = 1, MATCH_BAD_ORDER = 2, MATCH_BAD_LAST = 4;

// q_off[0] == 0, ascending, q_off[nq] == q_bytes
__global__ void __launch_bounds__(BLK) k_match_check(const uint64_t *__restrict__ qoff, uint32_t nq, uint64_t q_bytes,
                                                     uint32_t *word) {
    uint64_t q = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    uint32_t bad = 0;
    if (q <= nq) {
        const uint64_t v = qoff[q];
        if (q == 0 && v != 0) bad |= MATCH_BAD_FIRST;
        if (q < nq && qoff[q + 1] < v) bad |= MATCH_BAD_ORDER;
        if (q == nq && v != q_bytes) bad |= MATCH_BAD_LAST;
    }
    bad = __reduce_or_sync(FULL, bad);
    if (bad && lane_id() == 0) atomicOr(word, bad);
}

// the query of pattern position x: the last q with q_off[q] <= x (an empty query shares its offset
// with the next one, so x lands in the non-empty one)
__device__ __forceinline__ uint32_t match_query_of(const uint64_t *__restrict__ qoff, uint32_t nq, uint64_t x) {
    uint32_t a = 0, b = nq;
    while (b - a > 1) {
        uint32_t m = a + (b - a) / 2;
        if (__ldg(qoff + m) <= x) a = m; else b = m;
    }
    return a;
}

// A caller's byte buffer and the offsets [lo, hi) of the 4-byte words that lie wholly inside it: the
// compare loads whole aligned words only there, and single bytes elsewhere, so it never touches a byte
// outside the buffer whatever the alignment of its base.
struct MatchBuf {
    const uint8_t *base;
    long long lo, hi;
    __host__ MatchBuf(const uint8_t *b, uint64_t len) : base(b) {
        const uint64_t a = (uint64_t)(uintptr_t)b;
        lo = (long long)((4 - (a & 3)) & 3);
        hi = (long long)(((a + len) & ~(uint64_t)3) - a);   // below lo when the buffer holds no whole word
    }
};

// Extends c, the known common prefix of the pattern Q[x, x + m) and the suffix T[p, p + ls), to its full
// length.  *lt = the pattern's byte is below the suffix's where they first differ (false if a side ends).
// Word steps: 4 bytes of either side are the funnel shift of two aligned words, the second one carried
// into the next step; the first differing byte is the lowest set byte of the XOR (little endian).
__device__ __forceinline__ uint32_t match_extend(const MatchBuf &T, uint32_t p, uint32_t ls, const MatchBuf &Q,
                                                 uint64_t x, uint32_t m, uint32_t c, bool *lt) {
    const uint32_t l = ls < m ? ls : m;
    const uint8_t *t = T.base + p, *q = Q.base + x;
    *lt = false;
    // a step at c reads the words covering [c, c + 8) of both sides
    long long kend = (long long)l - 4;
    kend = min(kend, min(T.hi - 8 - (long long)p, Q.hi - 8 - (long long)x));
    const long long head = max(T.lo - (long long)p, Q.lo - (long long)x);   // > 0 only in a misaligned buffer's first word
    for (; c < l && (long long)c < head; c++) {
        const uint32_t a = q[c], b = __ldg(t + c);
        if (a != b) { *lt = a < b; return c; }
    }
    if ((long long)c <= kend) {
        const uintptr_t ta = (uintptr_t)(t + c), qa = (uintptr_t)(q + c);
        const uint32_t *tw = reinterpret_cast<const uint32_t *>(ta & ~(uintptr_t)3);
        const uint32_t *qw = reinterpret_cast<const uint32_t *>(qa & ~(uintptr_t)3);
        const uint32_t tsh = (uint32_t)(ta & 3) * 8, qsh = (uint32_t)(qa & 3) * 8;
        uint32_t t0 = __ldg(tw), q0 = __ldg(qw);
        do {
            const uint32_t t1 = __ldg(++tw), q1 = __ldg(++qw);
            const uint32_t b = __funnelshift_r(t0, t1, tsh), a = __funnelshift_r(q0, q1, qsh);
            const uint32_t d = a ^ b;
            if (d) {
                const uint32_t j = (__ffs(d) - 1) & ~7u;
                *lt = ((a >> j) & 0xffu) < ((b >> j) & 0xffu);
                return c + (j >> 3);
            }
            c += 4;
            t0 = t1;
            q0 = q1;
        } while ((long long)c <= kend);
    }
    for (; c < l; c++) {
        const uint32_t a = q[c], b = __ldg(t + c);
        if (a != b) { *lt = a < b; return c; }
    }
    return c;
}

// One thread per pattern position.  RANGE = false writes len alone (L, out_start and out_end unused).
template <class EndF, bool RANGE>
__global__ void __launch_bounds__(BLK) k_match_stats(MatchBuf T, uint32_t n, const uint32_t *__restrict__ sa,
                                                     AnsvLevels L, MatchBuf Q, const uint64_t *__restrict__ qoff,
                                                     uint32_t nq, uint64_t q_bytes, uint32_t *out_len,
                                                     uint32_t *out_start, uint32_t *out_end, EndF end) {
    const uint64_t x = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (x >= q_bytes) return;
    const uint32_t m = (uint32_t)(__ldg(qoff + match_query_of(qoff, nq, x) + 1) - x);
    uint32_t lo = 0, hi = n;                              // lo = the lower bound's rank + 1
    uint32_t llo = 0, lhi = 0, len = 0, w = 0;
    bool whole = false;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2, p = sa[mid], ls = end(p) - p;
        bool lt;
        const uint32_t c = match_extend(T, p, ls, Q, x, m, llo < lhi ? llo : lhi, &lt);
        if (c == m) {                                     // the whole rest of the query occurs
            whole = true;
            len = m;
            w = mid;
            break;
        }
        if (c < ls && lt) { hi = mid; lhi = c; } else { lo = mid + 1; llo = c; }
    }
    if (!whole) {
        len = llo >= lhi ? llo : lhi;
        w = llo >= lhi ? lo - 1 : hi;                     // a real rank whenever len > 0
    }
    out_len[x] = len;
    if (RANGE) {
        uint32_t s = 0, e = 0;
        if (len > 0) {
            s = L.lv[0][w] < len ? w : ansv_left<true>(L, w, len);   // lcp[0] = 0 < len: found
            e = (uint32_t)ansv_right(L, w, len, n);
        }
        out_start[x] = s;
        out_end[x] = e;
    }
}

// Super-maximal exact matches: position x of query q with len[x] >= min_len and (x is q's first byte or
// len[x - 1] <= len[x]).  x + len[x] never decreases inside a query, so these are the matches
// [x, x + len[x]) that no other match of the query contains.  Entry q_bytes is 0 (the scan's total slot).
__global__ void __launch_bounds__(BLK) k_smem_flag(const uint32_t *__restrict__ len, const uint64_t *__restrict__ qoff,
                                                   uint32_t nq, uint64_t q_bytes, uint32_t min_len, uint32_t *flag) {
    const uint64_t x = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (x > q_bytes) return;
    uint32_t f = 0;
    if (x < q_bytes) {
        const uint32_t v = len[x];
        if (v >= min_len) f = (x == 0 || len[x - 1] <= v || __ldg(qoff + match_query_of(qoff, nq, x)) == x) ? 1u : 0u;
    }
    flag[x] = f;
}
struct SmemIn {
    const uint32_t *flag;
    __device__ uint32_t operator()(uint64_t i) const { return flag[i]; }
};
struct SmemOut {
    uint32_t *exc;
    __device__ void operator()(uint64_t i, uint32_t e, uint32_t) const { exc[i] = e; }
};
// offsets[q] = the flagged positions before q's first byte; with qpos, the flagged positions compacted in
// ascending x as offsets inside their query.
__global__ void __launch_bounds__(BLK) k_smem_emit(const uint32_t *__restrict__ flag, const uint32_t *__restrict__ exc,
                                                   const uint64_t *__restrict__ qoff, uint32_t nq, uint64_t q_bytes,
                                                   unsigned long long *offsets, uint32_t *qpos) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i <= nq) offsets[i] = exc[qoff[i]];
    if (qpos && i < q_bytes && flag[i]) qpos[exc[i]] = (uint32_t)(i - __ldg(qoff + match_query_of(qoff, nq, i)));
}

}  // namespace b200sa
