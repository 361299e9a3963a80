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
// Slot ranges are cut into chunks of 1024 ranks numbered by a u64 scan (DListChunks), as the listing of
// docs_list.cuh cuts its ranges; one warp walks one (slot, chunk) item (approx_item), one rank per lane per
// step.  A count pass, a scan, k_dlist_qoff with a stride of P slots, then an emit pass of the same walk that
// writes (q, p) keys in item order, sorted afterwards.
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

// The (slot, chunk) item a warp walks: query q of m bytes at qq, its piece j at offset oj (0 in the whole-table
// slot, whole) and the ranks [lo, hi) of the slot's range in the chunk.
struct ApproxItem {
    uint32_t q, j, m, oj;
    bool whole;
    const uint8_t *qq;
    uint64_t lo, hi;
};
template <class Pieces>
__device__ __forceinline__ ApproxItem approx_item(const ApproxArgs &A, uint64_t item) {
    const DListItem it = dlist_item(A.item_start, A.nslots, A.ps, A.pe, item);
    const uint32_t q = it.r / A.P, j = it.r % A.P;
    const uint64_t qo = A.qoff[q];
    const uint32_t m = (uint32_t)(A.qoff[q + 1] - qo);
    const bool whole = Pieces::whole(A, it.r, m);
    return {q, j, m, whole ? 0u : Pieces::off(A, it.r, m, j), whole, A.qs + qo, it.lo, it.hi};
}

// The document [*ds, *de) that holds position s, or the text [0, n)
__device__ __forceinline__ void approx_doc(const ApproxArgs &A, uint32_t s, uint32_t *ds, uint32_t *de) {
    *ds = 0;
    *de = A.n;
    if (A.starts) {
        const uint32_t d = docs_find(A.starts, A.ndocs, s);
        *ds = __ldg(A.starts + d);
        *de = docs_end(A.starts, A.ndocs, A.n, d);
    }
}

// Whether the piece bytes pq[0, len) are the text's at t
__device__ __forceinline__ bool approx_piece_at(const uint8_t *__restrict__ t, const uint8_t *__restrict__ pq,
                                                uint32_t len) {
    for (uint32_t y = 0; y < len; y++)
        if (__ldg(t + y) != __ldg(pq + y)) return false;
    return true;
}

// The pieces [a, b) of a query of m bytes in order, piece i = [i*m/P, (i+1)*m/P): next() steps to the following
// piece by m/P and the remainder m%P, with no division per piece.
struct CutStep {
    uint32_t P, step, rem, a = 0, b = 0, r = 0;
    __device__ __forceinline__ CutStep(uint32_t m, uint32_t P) : P(P), step(m / P), rem(m % P) {}
    __device__ __forceinline__ void next() {
        a = b;
        b += step;
        r += rem;
        if (r >= P) { b++; r -= P; }
    }
};

// The pieces of a query, as a policy of the walks of k_approx (verify) and k_approx_edit (CLASSES, whole_hits,
// reports, FIXED): f-14's pieces and byte equality here, the piece table and the class test (miss) of IupacPieces
// and FixedIupacPieces (iupac.cuh).  whole(slot, m): whether the slot is the whole table; off: the offset of piece j.
struct CutPieces {
    static __device__ __forceinline__ bool whole(const ApproxArgs &A, uint32_t, uint32_t m) { return m <= A.k; }
    static __device__ __forceinline__ uint32_t off(const ApproxArgs &A, uint32_t, uint32_t m, uint32_t j) {
        return approx_cut(m, A.P, j);
    }
    // (offset, length) of piece i of query q of m bytes
    static __device__ __forceinline__ uint2 piece(const ApproxArgs &A, uint32_t, uint32_t m, uint32_t i) {
        const uint32_t a = approx_cut(m, A.P, i);
        return make_uint2(a, approx_cut(m, A.P, i + 1) - a);
    }
    // Whether the suffix at s, a candidate of the item's slot, starts an occurrence this slot reports; then
    // *p_out = its position and *mis_out = its mismatches.
    static __device__ __forceinline__ bool verify(const ApproxArgs &A, const ApproxItem &w, uint32_t s,
                                                  uint32_t *p_out, uint32_t *mis_out) {
        if (s < w.oj) return false;
        const uint32_t p = s - w.oj;
        uint32_t ds, de;
        approx_doc(A, s, &ds, &de);
        if (p < ds || (uint64_t)p + w.m > de) return false;
        const uint8_t *__restrict__ t = A.text + p;
        const uint8_t *__restrict__ qq = w.qq;
        uint32_t mis = 0;
        if (w.whole) {
            for (uint32_t x = 0; x < w.m; x++) mis += __ldg(t + x) != __ldg(qq + x);
        } else {
            CutStep pc(w.m, A.P);
            for (uint32_t i = 0; i < A.P; i++) {
                pc.next();
                if (i == w.j) continue;
                uint32_t mi = 0;
                for (uint32_t x = pc.a; x < pc.b && mis + mi <= A.k; x++) mi += __ldg(t + x) != __ldg(qq + x);
                if (i < w.j && mi == 0) return false;        // slot i reports it
                mis += mi;
                if (mis > A.k) return false;
            }
        }
        *p_out = p;
        *mis_out = mis;
        return true;
    }
    static constexpr bool CLASSES = false;      // byte equality, which edit_verify tests inline
    static constexpr bool FIXED = false;        // every query symbol may take an edit
    // dist(s) <= m <= k in the whole-table slot
    static __device__ __forceinline__ uint64_t whole_hits(const uint8_t *, int32_t k) { return 1ull << k; }
    static __device__ __noinline__ bool reports(const ApproxArgs &A, int64_t p, uint32_t s,
                                                const uint8_t *__restrict__ qq, uint32_t m, uint32_t q, uint32_t j,
                                                uint32_t oj, uint32_t ds, uint32_t de);     // edit.cuh
};

// EMIT = false: cnt[item] = the occurrences the item reports.  EMIT = true: the same walk writes them from
// item_off[item] on, in rank order: key = (q << pbits) | p, val = mis(p).
template <bool EMIT, class Pieces>
__device__ __forceinline__ void approx_walk(ApproxArgs A, uint32_t *cnt, const unsigned long long *item_off, int pbits,
                                            unsigned long long *key, uint32_t *val) {
    const uint64_t item = ((uint64_t)blockIdx.x * BLK + threadIdx.x) >> 5;
    if (item >= A.items) return;                                  // whole warps
    const uint32_t l = lane_id();
    const ApproxItem w = approx_item<Pieces>(A, item);
    const uint64_t base = EMIT ? item_off[item] : 0;
    uint32_t count = 0;
    for (uint64_t i0 = w.lo; i0 < w.hi; i0 += 32) {               // the same trip count on every lane
        const uint64_t i = i0 + l;
        uint32_t p = 0, mis = 0;
        const bool hit = i < w.hi && Pieces::verify(A, w, A.sa[i], &p, &mis);
        const uint32_t m0 = __ballot_sync(FULL, hit);
        if (EMIT && hit) {
            const uint64_t slot = base + count + __popc(m0 & lanemask_lt());
            key[slot] = ((unsigned long long)w.q << pbits) | p;
            val[slot] = mis;
        }
        count += __popc(m0);
    }
    if (!EMIT && l == 0) cnt[item] = count;
}

template <bool EMIT>
__global__ void __launch_bounds__(BLK) k_approx(ApproxArgs A, uint32_t *cnt, const unsigned long long *item_off,
                                                int pbits, unsigned long long *key, uint32_t *val) {
    approx_walk<EMIT, CutPieces>(A, cnt, item_off, pbits, key, val);
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
