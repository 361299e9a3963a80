// approx.cuh -- every occurrence of each query with at most k substituted bytes (DESIGN 6b f-14).
//
// Pigeonhole filter, then verification (the partition lemma of Wu & Manber 1992 and Baeza-Yates &
// Perleberg 1996).  A query of m > k bytes is cut into P = k + 1 pieces, piece j = [j*m/P, (j+1)*m/P), all
// non-empty; a window with at most k mismatches matches at least one piece exactly.  Slot (q, j), at
// q*P + j, holds the range of the table whose suffixes start with piece j (positions_range).  A query of
// 0 < m <= k has one slot, j = 0, holding the whole table [0, n) with an empty piece at offset 0: every
// window of m bytes qualifies.  m = 0 has no slot range.
// A candidate of slot (q, j) is a rank i, s = R[i], p = s - o_j (o_j the piece's offset).  It is reported by
// that slot when the window [p, p + m) lies in s's document (the text), no piece i < j matches exactly
// there and the pieces other than j add at most k mismatches.  The first exactly matching piece is thus the
// one reporter of an occurrence: nothing is emitted twice and no de-duplication is needed.
// Slot ranges are cut into chunks of 1024 ranks numbered by a u64 scan (DListChunks); one warp walks one
// (slot, chunk) item, one rank per lane per step.  A count pass, a scan, then an emit pass of the same walk
// that writes (q, p) keys in item order, sorted afterwards.
#pragma once
#include "docs_list.cuh"

namespace b200sa {

// j*m/P, the offset of piece j of a query of m bytes
__device__ __forceinline__ uint32_t approx_cut(uint32_t m, uint32_t P, uint32_t j) {
    return (uint32_t)((uint64_t)j * m / P);
}

// The slot ranges: ps / pe[q*P + j] (one thread per slot; n >= 1).
template <class EndF>
__global__ void __launch_bounds__(BLK) k_approx_pieces(const uint8_t *__restrict__ text, uint32_t n,
                                                       const uint32_t *__restrict__ sa, const uint8_t *__restrict__ qs,
                                                       const uint64_t *__restrict__ qoff, uint32_t nq, uint32_t P,
                                                       uint32_t *ps, uint32_t *pe, EndF end) {
    const uint64_t slot = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (slot >= (uint64_t)nq * P) return;
    const uint32_t q = (uint32_t)(slot / P), j = (uint32_t)(slot % P);
    const uint64_t o = qoff[q];
    const uint32_t m = (uint32_t)(qoff[q + 1] - o);
    uint32_t s = 0, e = 0;
    if (m >= P) {
        const uint32_t a = approx_cut(m, P, j), b = approx_cut(m, P, j + 1);
        positions_range(text, n, sa, qs + o + a, b - a, end, &s, &e);
    } else if (m > 0 && j == 0) {
        e = n;
    }
    ps[slot] = s;
    pe[slot] = e;
}

struct ApproxArgs {
    const uint8_t *text;
    const uint32_t *sa;
    const uint32_t *starts;                  // doc_starts, or NULL for a single text
    uint32_t ndocs, n;
    const uint8_t *qs;
    const uint64_t *qoff;
    uint32_t nslots, P, k;                   // nslots = nq * P, P = k + 1
    const uint32_t *ps, *pe;                 // the slot ranges
    const unsigned long long *item_start;    // [nslots + 1]: first item of each slot
    uint64_t items;
};

// Whether the suffix at s, a candidate of piece j at offset oj of the query qq of m bytes, starts an
// occurrence this slot reports; then *p_out = its position and *mis_out = its mismatches.  whole: m <= k.
__device__ __forceinline__ bool approx_verify(const ApproxArgs &A, uint32_t s, const uint8_t *__restrict__ qq,
                                              uint32_t m, uint32_t j, uint32_t oj, bool whole, uint32_t *p_out,
                                              uint32_t *mis_out) {
    if (s < oj) return false;
    const uint32_t p = s - oj;
    uint32_t ds = 0, de = A.n;
    if (A.starts) {
        const uint32_t d = docs_find(A.starts, A.ndocs, s);
        ds = __ldg(A.starts + d);
        de = docs_end(A.starts, A.ndocs, A.n, d);
    }
    if (p < ds || (uint64_t)p + m > de) return false;
    const uint8_t *__restrict__ t = A.text + p;
    uint32_t mis = 0;
    if (whole) {
        for (uint32_t x = 0; x < m; x++) mis += __ldg(t + x) != __ldg(qq + x);
    } else {
        // piece i = [a, b) with a = i*m/P, stepped by m/P and the remainder m%P
        const uint32_t step = m / A.P, rem = m % A.P;
        uint32_t a = 0, r = 0;
        for (uint32_t i = 0; i < A.P; i++) {
            uint32_t b = a + step;
            r += rem;
            if (r >= A.P) { b++; r -= A.P; }
            if (i != j) {
                uint32_t mi = 0;
                for (uint32_t x = a; x < b && mis + mi <= A.k; x++) mi += __ldg(t + x) != __ldg(qq + x);
                if (i < j && mi == 0) return false;          // slot i reports it
                mis += mi;
                if (mis > A.k) return false;
            }
            a = b;
        }
    }
    *p_out = p;
    *mis_out = mis;
    return true;
}

// f-14's pieces: piece j = [j*m/P, (j+1)*m/P), a whole-table slot for m <= k, and approx_verify.  The walks
// of k_approx and k_approx_edit take the pieces as a policy, so that B200SA_APPROX_IUPAC (iupac.cuh) reuses them.
struct CutPieces {
    __device__ __forceinline__ bool whole(const ApproxArgs &A, uint32_t, uint32_t m) const { return m <= A.k; }
    __device__ __forceinline__ uint32_t off(const ApproxArgs &A, uint32_t, uint32_t m, uint32_t j) const {
        return approx_cut(m, A.P, j);
    }
    __device__ __forceinline__ bool verify(const ApproxArgs &A, uint32_t s, const uint8_t *__restrict__ qq, uint32_t m,
                                           uint32_t, uint32_t j, uint32_t oj, bool whole, uint32_t *p_out,
                                           uint32_t *mis_out) const {
        return approx_verify(A, s, qq, m, j, oj, whole, p_out, mis_out);
    }
};

// EMIT = false: cnt[item] = the occurrences the item reports.  EMIT = true: the same walk writes them from
// item_off[item] on, in rank order: key = (q << pbits) | p, val = mis(p).
template <bool EMIT, class Pieces>
__device__ __forceinline__ void approx_walk(ApproxArgs A, Pieces pc, uint32_t *cnt,
                                            const unsigned long long *item_off, int pbits, unsigned long long *key,
                                            uint32_t *val) {
    const uint64_t item = ((uint64_t)blockIdx.x * BLK + threadIdx.x) >> 5;
    if (item >= A.items) return;                                  // whole warps
    const uint32_t l = lane_id();
    uint32_t a = 0, b = A.nslots;                                 // the last slot whose first item <= item
    while (b - a > 1) {
        const uint32_t mid = a + (b - a) / 2;
        if (A.item_start[mid] <= item) a = mid; else b = mid;
    }
    const uint32_t q = a / A.P, j = a % A.P;
    const uint32_t s0 = A.ps[a], e0 = A.pe[a];
    const uint64_t blk = s0 / DLIST_CHUNK + (item - A.item_start[a]);
    const uint64_t lo = blk * DLIST_CHUNK > s0 ? blk * DLIST_CHUNK : s0;
    const uint64_t hi = blk * DLIST_CHUNK + DLIST_CHUNK < e0 ? blk * DLIST_CHUNK + DLIST_CHUNK : e0;
    const uint64_t qo = A.qoff[q];
    const uint32_t m = (uint32_t)(A.qoff[q + 1] - qo);
    const bool whole = pc.whole(A, a, m);
    const uint32_t oj = whole ? 0u : pc.off(A, a, m, j);
    const uint64_t base = EMIT ? item_off[item] : 0;
    uint32_t count = 0;
    for (uint64_t i0 = lo; i0 < hi; i0 += 32) {                   // the same trip count on every lane
        const uint64_t i = i0 + l;
        uint32_t p = 0, mis = 0;
        const bool hit = i < hi && pc.verify(A, A.sa[i], A.qs + qo, m, q, j, oj, whole, &p, &mis);
        const uint32_t m0 = __ballot_sync(FULL, hit);
        if (EMIT && hit) {
            const uint64_t slot = base + count + __popc(m0 & lanemask_lt());
            key[slot] = ((unsigned long long)q << pbits) | p;
            val[slot] = mis;
        }
        count += __popc(m0);
    }
    if (!EMIT && l == 0) cnt[item] = count;
}

template <bool EMIT>
__global__ void __launch_bounds__(BLK) k_approx(ApproxArgs A, uint32_t *cnt, const unsigned long long *item_off,
                                                int pbits, unsigned long long *key, uint32_t *val) {
    approx_walk<EMIT>(A, CutPieces{}, cnt, item_off, pbits, key, val);
}

// offsets[q] = the output offset of query q's first item (its slots are q*P .. q*P + P - 1)
__global__ void __launch_bounds__(BLK) k_approx_qoff(const unsigned long long *__restrict__ item_start,
                                                     const unsigned long long *__restrict__ item_off, uint32_t nq,
                                                     uint32_t P, unsigned long long *offsets) {
    const uint64_t q = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (q > nq) return;
    offsets[q] = item_off[item_start[q * P]];
}

// The sorted keys and values into the caller's arrays (mis may be NULL).
__global__ void __launch_bounds__(BLK) k_approx_gather(const unsigned long long *__restrict__ key,
                                                       const uint32_t *__restrict__ val, uint64_t total,
                                                       unsigned long long pmask, uint32_t *pos, uint32_t *mis) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= total) return;
    pos[i] = (uint32_t)(key[i] & pmask);
    if (mis) mis[i] = val[i];
}

}  // namespace b200sa
