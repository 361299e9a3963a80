// repeats.cuh -- what in the text repeats itself (DESIGN 6b f-11): the repeat length of every position,
// the runs of the table at a length L (the distinct L-byte strings that occur at least twice) and the
// spans of bytes covered by repeated L-grams.
//
// R is the table (sa or G), lam(i) its LCP array with lam(n) = 0.  Rank r is *in a run* at L when
// lam(r) >= L or lam(r + 1) >= L.  The ranks r with lam(r) < L cut the table into segments: a run is a
// segment of two or more ranks, every other rank a segment of one.  seg[r] is the rank of r's segment
// head, a max scan of (lam(r) < L ? r + 1 : 0).
//
// The smallest (largest) position of every segment is ONE inclusive max scan of the 64-bit key
// (seg[r] << 32 | value): seg never decreases with r, so the maximum over [0, r] is attained inside r's own
// segment and its low word is the segment's maximum so far.  The scan operator stays a plain max --
// commutative, as k_scan_lb's warp and look-back reductions require; a (head bit, value) operator is
// not -- and the value read at the segment's last rank is that of the whole segment, however long it is
// and however many tiles it crosses.  first = min position scans ~position, last scans the position.
#pragma once
#include "docs.cuh"

namespace b200sa {

struct OpMax64 {
    using T = unsigned long long;
    __device__ __forceinline__ static T id() { return 0ull; }
    __device__ __forceinline__ static T op(T a, T b) { return a > b ? a : b; }
};

// lam(i) for i in [0, n]
__device__ __forceinline__ uint32_t rep_lam(const uint32_t *__restrict__ lcp, uint32_t n, uint64_t i) {
    return i < n ? lcp[i] : 0u;
}

// rl[R[r]] = max(lam(r), lam(r + 1))
__global__ void __launch_bounds__(BLK) k_rep_lens(const uint32_t *__restrict__ sa, const uint32_t *__restrict__ lcp,
                                                  uint32_t n, uint32_t *rl) {
    const uint64_t r = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (r >= n) return;
    const uint32_t a = lcp[r], b = rep_lam(lcp, n, r + 1);
    rl[sa[r]] = a > b ? a : b;
}

// ---- runs: 1 at the first rank of every run
struct RepRunIn {
    const uint32_t *lcp;
    uint32_t n, L;
    __device__ uint32_t operator()(uint64_t r) const { return (lcp[r] < L && rep_lam(lcp, n, r + 1) >= L) ? 1u : 0u; }
};
struct RepNoOut {
    __device__ void operator()(uint64_t, uint32_t, uint32_t) const {}
};
// start at the run's first rank (run index = exclusive count), end at its last (inclusive count - 1, and
// a last rank is never a first one); first / last are read at the segment head
struct RepRunOut {
    const uint32_t *lcp;
    uint32_t n, L;
    uint32_t *start, *end, *first, *last;
    const uint32_t *seg_first, *seg_last;
    __device__ void operator()(uint64_t r, uint32_t exc, uint32_t head) const {
        if (head) {
            start[exc] = (uint32_t)r;
            if (first) first[exc] = seg_first[r];
            if (last) last[exc] = seg_last[r];
        } else if (lcp[r] >= L && rep_lam(lcp, n, r + 1) < L) {
            end[exc - 1] = (uint32_t)r + 1;
        }
    }
};

// ---- segments
struct RepSegIn {
    const uint32_t *lcp;
    uint32_t L;
    __device__ uint32_t operator()(uint64_t r) const { return lcp[r] < L ? (uint32_t)r + 1 : 0u; }
};
struct RepSegOut {                      // lam(0) = 0 < L: the inclusive maximum is at least 1
    uint32_t *seg;
    __device__ void operator()(uint64_t r, uint32_t exc, uint32_t v) const { seg[r] = (exc > v ? exc : v) - 1; }
};
// NEG: the smallest position (the key carries ~position), else the largest
template <bool NEG>
struct RepExtIn {
    const uint32_t *sa, *seg;
    __device__ unsigned long long operator()(uint64_t r) const {
        const uint32_t p = sa[r];
        return ((unsigned long long)seg[r] << 32) | (NEG ? ~p : p);
    }
};
template <bool NEG>
struct RepExtOut {                      // written at the segment's last rank, to the slot of its head
    const uint32_t *lcp;
    uint32_t n, L;
    uint32_t *seg_ext;
    __device__ void operator()(uint64_t r, unsigned long long exc, unsigned long long v) const {
        if (rep_lam(lcp, n, r + 1) < L) {
            const unsigned long long m = exc > v ? exc : v;
            seg_ext[(uint32_t)(v >> 32)] = NEG ? ~(uint32_t)m : (uint32_t)m;
        }
    }
};

// ---- flagged positions, one thread per rank; only flagged positions are written (bits of a zeroed bitmap)
enum { REP_ANY = 0, REP_EARLIER = 1, REP_OTHER_DOC = 2, REP_EARLIER_DOC = 3 };
template <int MODE>
__global__ void __launch_bounds__(BLK) k_rep_flag(const uint32_t *__restrict__ sa, const uint32_t *__restrict__ lcp,
                                                  uint32_t n, uint32_t L, const uint32_t *__restrict__ seg,
                                                  const uint32_t *__restrict__ seg_first,
                                                  const uint32_t *__restrict__ seg_last,
                                                  const uint32_t *__restrict__ starts, uint32_t ndocs, uint32_t *bits) {
    const uint64_t r = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (r >= n) return;
    if (lcp[r] < L && rep_lam(lcp, n, r + 1) < L) return;          // in no run
    const uint32_t p = sa[r];
    bool f = true;
    if (MODE == REP_EARLIER) {
        f = p != seg_first[seg[r]];
    } else if (MODE == REP_OTHER_DOC || MODE == REP_EARLIER_DOC) {
        const uint32_t h = seg[r], d = docs_find(starts, ndocs, p);
        f = seg_first[h] < __ldg(starts + d);
        if (MODE == REP_OTHER_DOC) f = f || seg_last[h] >= docs_end(starts, ndocs, n, d);
    }
    if (f) atomicOr(bits + (p >> 5), 1u << (p & 31));
}

// document starts inside (0, n), one thread per document
__global__ void __launch_bounds__(BLK) k_rep_doc_bits(const uint32_t *__restrict__ starts, uint32_t ndocs, uint32_t n,
                                                      uint32_t *bits) {
    const uint32_t d = blockIdx.x * BLK + threadIdx.x;
    if (d >= ndocs) return;
    const uint32_t s = starts[d];
    if (s > 0 && s < n) atomicOr(bits + (s >> 5), 1u << (s & 31));
}

// ---- cover, in text order: near[x] = 1 + the last flagged position at or before x (0: none)
__device__ __forceinline__ bool rep_bit(const uint32_t *__restrict__ bits, uint64_t x) {
    return (bits[x >> 5] >> (x & 31)) & 1u;
}
struct RepNearIn {
    const uint32_t *bits;
    __device__ uint32_t operator()(uint64_t x) const { return rep_bit(bits, x) ? (uint32_t)x + 1 : 0u; }
};
struct RepNearOut {
    uint32_t *near;
    __device__ void operator()(uint64_t x, uint32_t exc, uint32_t v) const { near[x] = exc > v ? exc : v; }
};
// x is covered iff a flagged p has p <= x < p + L; the nearest such p decides
struct RepCover {
    const uint32_t *near, *doc_bits;
    uint32_t n, L;
    __device__ bool covered(uint64_t x) const {
        const uint32_t m = near[x];
        return m != 0 && (uint32_t)x - (m - 1) < L;
    }
    // a span begins at a covered byte whose predecessor is uncovered or that starts a document
    __device__ bool begins(uint64_t x) const { return x == 0 || rep_bit(doc_bits, x) || !covered(x - 1); }
    // ... and ends after a covered byte whose successor is uncovered or starts a document
    __device__ bool ends(uint64_t x) const { return x + 1 == n || rep_bit(doc_bits, x + 1) || !covered(x + 1); }
};
// high word: spans that begin at x; low word: x is covered.  Both sums stay below 2^32.
struct RepSpanIn {
    RepCover C;
    __device__ unsigned long long operator()(uint64_t x) const {
        if (!C.covered(x)) return 0ull;
        return ((unsigned long long)(C.begins(x) ? 1u : 0u) << 32) | 1ull;
    }
};
struct RepSpanNoOut {
    __device__ void operator()(uint64_t, unsigned long long, unsigned long long) const {}
};
struct RepSpanOut {
    RepCover C;
    uint32_t *begin, *end;
    __device__ void operator()(uint64_t x, unsigned long long exc, unsigned long long v) const {
        if (!v) return;
        const uint32_t k = (uint32_t)((exc + v) >> 32) - 1;         // the span x lies in
        if (v >> 32) begin[k] = (uint32_t)x;
        if (C.ends(x)) end[k] = (uint32_t)x + 1;
    }
};

}  // namespace b200sa
