// strand.cuh -- approximate occurrences on both DNA strands (DESIGN 6b f-18), the B200SA_APPROX_BOTH_STRANDS flag
// of the approximate-positions entry points.
//
// k_strand_queries writes the doubled batch: entry 2q is query q and entry 2q + 1 its reverse complement rc(q),
// both at twice q's byte offset, so the two strands of q are adjacent.  The search of approx.cuh / edit.cuh /
// iupac.cuh runs on it unchanged, and its sort orders the keys by (entry, p) = (2q + strand, p).  Entry 2q's first
// output is then q's first output, and k_strand_merge moves each hit to its place in q's list ordered by
// (p, strand): its index in its own sublist plus the number of hits of the other sublist before it, found by a
// binary search there.  With B200SA_APPROX_BEST the pair is the unit of liveness: StrandPick picks both entries of
// a live pair, k_strand_update keeps one best per pair, each emitted group scatters into a staging copy laid out
// over the doubled offsets, and one k_strand_merge reads that copy.
#pragma once
#include "best.cuh"

namespace b200sa {

// The complement of a query byte: A <-> T and C <-> G in either case, every other byte itself.  canon: a byte of
// iupac.cuh's canonical copy, whose concrete bases are uppercase and whose classes are masks A 1, C 2, G 4, T 8,
// so the complement of a class is its mask with the 4 bits reversed.
__device__ __forceinline__ uint32_t strand_comp(uint32_t b, bool canon) {
    if (canon && b < 16) return (b & 1) << 3 | (b & 2) << 1 | (b & 4) >> 1 | (b & 8) >> 3;
    switch (b) {
    case 'A': return 'T';
    case 'T': return 'A';
    case 'C': return 'G';
    case 'G': return 'C';
    case 'a': return 't';
    case 't': return 'a';
    case 'c': return 'g';
    case 'g': return 'c';
    default: return b;
    }
}

// The doubled batch of nq queries: out[2 qoff[q], + m) = q, then rc(q); qoff2[2q] = 2 qoff[q],
// qoff2[2q + 1] = 2 qoff[q] + m, qoff2[2 nq] = 2 qoff[nq].  One warp per query.
__global__ void __launch_bounds__(BLK) k_strand_queries(const uint8_t *__restrict__ qs,
                                                        const uint64_t *__restrict__ qoff, uint32_t nq, bool canon,
                                                        uint8_t *out, uint64_t *qoff2) {
    const uint64_t q = ((uint64_t)blockIdx.x * BLK + threadIdx.x) >> 5;
    if (q >= nq) return;
    const uint32_t l = lane_id();
    const uint64_t o = qoff[q], m = qoff[q + 1] - o;
    const uint8_t *__restrict__ src = qs + o;
    uint8_t *fw = out + 2 * o, *rc = fw + m;
    for (uint64_t x = l; x < m; x += 32) {
        fw[x] = src[x];
        rc[x] = (uint8_t)strand_comp(src[m - 1 - x], canon);
    }
    if (l == 0) {
        qoff2[2 * q] = 2 * o;
        qoff2[2 * q + 1] = 2 * o + m;
        if (q == nq - 1) qoff2[2 * q + 2] = 2 * (o + m);
    }
}

// The sorted hits of the search over the doubled batch: keys (entry << pbits) | p.
struct StrandKeys {
    const unsigned long long *key;
    int pbits;
    __device__ __forceinline__ uint32_t entry(uint64_t i, const unsigned long long *, uint32_t) const {
        return (uint32_t)(key[i] >> pbits);
    }
    __device__ __forceinline__ uint32_t pos(uint64_t i) const { return (uint32_t)(key[i] & ((1ull << pbits) - 1)); }
};
// The staging copy of B200SA_APPROX_BEST: positions laid out over the doubled offsets, each sublist ascending.
struct StrandStaged {
    const uint32_t *p;
    __device__ __forceinline__ uint32_t entry(uint64_t i, const unsigned long long *doff, uint32_t ne) const {
        uint32_t a = 0, b = ne;                                   // the last entry whose first hit <= i
        while (b - a > 1) {
            const uint32_t mid = a + (b - a) / 2;
            if (doff[mid] <= i) a = mid; else b = mid;
        }
        return a;
    }
    __device__ __forceinline__ uint32_t pos(uint64_t i) const { return p[i]; }
};

// The total hits of the ne = 2 nq entries, at the doubled offsets doff, into the caller's arrays ordered by
// (p, strand) per query: a + hit goes after the - hits with a smaller p, a - hit after the + hits with a p at
// most as large.  val[i] is hit i's distance; mis (may be NULL) gets it with B200SA_APPROX_MINUS on a - hit.
template <class Src>
__global__ void __launch_bounds__(BLK) k_strand_merge(Src src, const uint32_t *__restrict__ val, uint64_t total,
                                                      const unsigned long long *__restrict__ doff, uint32_t ne,
                                                      uint32_t *pos, uint32_t *mis) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= total) return;
    const uint32_t e = src.entry(i, doff, ne), p = src.pos(i), minus = e & 1u;
    uint64_t a = doff[e ^ 1u], b = doff[(e ^ 1u) + 1];           // the first other hit after i's place
    while (a < b) {
        const uint64_t mid = a + (b - a) / 2;
        const uint32_t pm = src.pos(mid);
        if (pm < p || (minus && pm == p)) a = mid + 1; else b = mid;
    }
    const uint64_t dst = doff[e & ~1u] + (i - doff[e]) + (a - doff[e ^ 1u]);
    pos[dst] = p;
    if (mis) mis[dst] = val[i] | (minus ? B200SA_APPROX_MINUS : 0u);
}

// offsets[q] = doff[2q] for q <= nq: both strands of q start at its + entry.
__global__ void __launch_bounds__(BLK) k_strand_offsets(const unsigned long long *__restrict__ doff, uint32_t nq,
                                                        unsigned long long *offsets) {
    const uint64_t q = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (q <= nq) offsets[q] = doff[2 * q];
}

// BestPick over the ne entries of the doubled batch, with the best of entry e's pair at best[e >> 1]: both entries
// of a pair have the same m, so they are picked together and stay adjacent in the batch.
struct StrandPick {
    const uint64_t *qoff;
    const uint8_t *best;
    uint32_t ne, t, s, k;
    bool group;
    __device__ unsigned long long operator()(uint64_t e) const {
        if (e >= ne) return 0ull;
        const uint32_t m = (uint32_t)(qoff[e + 1] - qoff[e]), b = best[e >> 1];
        const bool in = group ? b != BEST_NONE && min(k, b + s) == t
                              : m > 0 && (b == BEST_NONE || t <= b + s);
        return in ? (1ull << 32) | m : 0ull;
    }
};

// k_best_update for pairs: batch entries 2i, 2i + 1 are the two strands of one query; cnt per entry, best per pair.
__global__ void __launch_bounds__(BLK) k_strand_update(const uint32_t *__restrict__ map,
                                                       const unsigned long long *__restrict__ roff, uint32_t nb,
                                                       uint32_t t, uint32_t s, uint32_t k, uint8_t *best,
                                                       uint32_t *cnt, uint32_t *ended) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= nb / 2) return;
    const uint32_t e = map[2 * i];
    const uint32_t c0 = (uint32_t)(roff[2 * i + 1] - roff[2 * i]), c1 = (uint32_t)(roff[2 * i + 2] - roff[2 * i + 1]);
    uint32_t b = best[e >> 1];
    cnt[e] = c0;
    cnt[e + 1] = c1;
    if (b == BEST_NONE && (c0 | c1)) best[e >> 1] = (uint8_t)(b = t);
    if (b != BEST_NONE && (t == k || t == b + s)) atomicOr(ended, 1u << t);
}

}  // namespace b200sa
