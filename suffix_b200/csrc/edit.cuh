// edit.cuh -- every occurrence of each query within k edits (DESIGN 6b f-15), the B200SA_APPROX_EDIT metric of
// the approximate-positions entry points.
//
// The partition lemma holds for Levenshtein distance too (Baeza-Yates & Navarro): an alignment of a query of
// m > k bytes with at most k edits leaves one of its P = k + 1 pieces matched exactly, shifted by at most k from
// its place in the query.  So the slots, chunks and count -> scan -> emit -> sort flow of approx.cuh carry over,
// and with them the item (approx_item), the document window (approx_doc) and the pieces (CutPieces); only the
// candidate's work differs.
// A candidate is a rank i of slot (q, j), s = R[i], c = s - o_j.  It considers the starts p of s's document
// [ds, de) with |p - c| <= k (at most 2k + 1 <= 63: one 64-bit mask per lane).  An alignment of cost <= k that
// starts at such a p stays within diagonals t - x in [c - 2k, c + 2k] (t a text, x a query position), so one
// reversed Sellers DP (query read backwards, text leftwards, a free end) over that band of 4k + 1 diagonals gives
// dist(p) exactly wherever it is <= k, for all of the window's starts at once.
// Reporter: R(p) is the least (i, s'') with piece i exactly at s'' inside p's document and |s'' - o_i - p| <= k;
// the candidate emits p iff dist(p) <= k and R(p) = (j, s) (the policy's reports).  The lemma makes R(p) exist
// for every occurrence, so each is emitted once, and the count pass is exact without de-duplication.
// A query of 0 < m <= k keeps the whole-table slot; there each rank reports its own position s with dist(s).
#pragma once
#include "approx.cuh"

namespace b200sa {

constexpr int EDIT_BAND = 4 * B200SA_APPROX_MAX_K + 1;    // diagonals of the widest band

// Whether piece bytes pq[0, len) occur at x, with [x, x + len) inside [ds, de)
__device__ __forceinline__ bool edit_piece_at(const uint8_t *__restrict__ text, int64_t x,
                                              const uint8_t *__restrict__ pq, uint32_t len, uint32_t ds, uint32_t de) {
    return x >= (int64_t)ds && x + len <= (int64_t)de && approx_piece_at(text + x, pq, len);
}

// Whether candidate (j, s) is R(p) for the start p of [ds, de): no piece i < j within k of its place, and no
// occurrence of piece j at s'' < s within k of its place.  Called only for starts within k; kept out of line,
// which keeps k_approx_edit<true> free of spills.
__device__ __noinline__ bool CutPieces::reports(const ApproxArgs &A, int64_t p, uint32_t s,
                                                const uint8_t *__restrict__ qq, uint32_t m, uint32_t, uint32_t j,
                                                uint32_t oj, uint32_t ds, uint32_t de) {
    const int32_t k = (int32_t)A.k;
    CutStep pc(m, A.P);
    for (uint32_t i = 0; i < j; i++) {
        pc.next();
        for (int32_t d = -k; d <= k; d++)
            if (edit_piece_at(A.text, p + pc.a + d, qq + pc.a, pc.b - pc.a, ds, de)) return false;
    }
    const uint32_t len = approx_cut(m, A.P, j + 1) - oj;
    for (int64_t x = p + oj - k; x < (int64_t)s; x++)
        if (edit_piece_at(A.text, x, qq + oj, len, ds, de)) return false;
    return true;
}

// The starts this candidate reports, bit b for p = c - k + b, with *c_out = c and v[k + b] = dist(p).  v holds
// one band row: v[d] = D(x, t) at t = c - 2k + x + d, D(x, t) = min over e of ED(q[x, m), T[t, e)), e <= de,
// saturated at k + 1.  whole: the whole-table slot, only p = s (o_j = 0).  Pieces: CutPieces, IupacPieces or
// FixedIupacPieces; with Pieces::FIXED a fixed q[x] is never substituted (X) or inserted (I), and no deleted text
// byte (D) sits next to one: no D at (x, t) when q[x] or q[x - 1] is fixed (DESIGN 6b f-21).
template <class Pieces>
__device__ __forceinline__ uint64_t edit_verify(const ApproxArgs &A, const ApproxItem &w, uint32_t s, uint8_t *v,
                                                int64_t *c_out) {
    const int32_t k = (int32_t)A.k, W = 4 * k + 1;
    const uint32_t INF = (uint32_t)k + 1;
    const uint8_t *__restrict__ qq = w.qq;
    const uint32_t m = w.m;
    uint32_t ds, de;
    approx_doc(A, s, &ds, &de);
    const int64_t c = (int64_t)s - w.oj, base = c - 2 * k;
    *c_out = c;
    for (int32_t d = 0; d < W; d++) {                      // row m: the empty rest of the query ends anywhere
        const int64_t t = base + m + d;
        v[d] = (t >= (int64_t)ds && t <= (int64_t)de) ? 0 : INF;
    }
    for (int64_t x = (int64_t)m - 1; x >= 0; x--) {        // in place, d downwards: v[d - 1] is still row x + 1
        const uint32_t qc = __ldg(qq + x);
        uint32_t right = INF, low = INF, old = v[W - 1];   // D(x, t + 1); the row's minimum; D(x + 1, t + 1)
        bool fx = false, nodel = false;                    // q[x] is fixed; the row has no D move
        if constexpr (Pieces::FIXED) {                     // q's marks, found again each row: one register less
            const uint8_t *__restrict__ mk = Pieces::marks(A, qq);
            fx = __ldg(mk + x) != 0;
            nodel = fx || (x > 0 && __ldg(mk + x - 1) != 0);
        }
        for (int32_t d = W - 1; d >= 0; d--) {
            const uint32_t up = d > 0 ? v[d - 1] : INF;    // D(x + 1, t)
            const int64_t t = base + x + d;
            uint32_t y = INF;
            if (t >= (int64_t)ds && t < (int64_t)de) {
                // the byte test written inline: through a miss() member, ptxas spends three predicate instructions
                // per unrolled cell where this spends one (8 more in k_approx_edit)
                if constexpr (Pieces::FIXED) {
                    const uint32_t mi = Pieces::miss(__ldg(A.text + t), qc);
                    y = min(nodel ? INF : right + 1, fx ? (mi ? INF : old) : min(up + 1, old + mi));
                } else if constexpr (Pieces::CLASSES) {
                    y = min(min(right, up) + 1, old + Pieces::miss(__ldg(A.text + t), qc));
                } else {
                    y = min(min(right, up) + 1, old + (__ldg(A.text + t) != qc));
                }
            } else if (t == (int64_t)de) {
                y = fx ? INF : up + 1;                     // no text left: delete q[x] (never a fixed one)
            }
            y = min(y, INF);
            v[d] = (uint8_t)y;
            right = y;
            low = min(low, y);
            old = up;
        }
        if (low > (uint32_t)k) return 0;                   // every path to row 0 passes this row
    }
    if (w.whole) return Pieces::whole_hits(v, k);
    const int64_t lo = max((int64_t)ds, c - k), hi = min((int64_t)de - 1, c + k);
    uint64_t hits = 0;
    for (int64_t p = lo; p <= hi; p++) {
        const uint32_t b = (uint32_t)(p - (c - k));
        if (v[k + b] <= (uint32_t)k && Pieces::reports(A, p, s, qq, m, w.q, w.j, w.oj, ds, de)) hits |= 1ull << b;
    }
    return hits;
}

// EMIT = false: cnt[item] = the occurrences the item reports.  EMIT = true: the same walk writes them from
// item_off[item] on: key = (q << pbits) | p, val = dist(p).  v: the kernel's band row of EDIT_BAND bytes.
template <bool EMIT, class Pieces>
__device__ __forceinline__ void edit_walk(ApproxArgs A, uint8_t *v, uint32_t *cnt, const unsigned long long *item_off,
                                          int pbits, unsigned long long *key, uint32_t *val) {
    const uint64_t item = ((uint64_t)blockIdx.x * BLK + threadIdx.x) >> 5;
    if (item >= A.items) return;                                  // whole warps
    const uint32_t l = lane_id();
    const ApproxItem w = approx_item<Pieces>(A, item);
    const uint64_t base = EMIT ? item_off[item] : 0;
    uint32_t count = 0;
    for (uint64_t i0 = w.lo; i0 < w.hi; i0 += 32) {               // the same trip count on every lane
        const uint64_t i = i0 + l;
        int64_t c = 0;
        const uint64_t hits = i < w.hi ? edit_verify<Pieces>(A, w, A.sa[i], v, &c) : 0;
        const uint32_t h = __popcll(hits);
        uint32_t incl = h;                                        // inclusive warp scan of the lanes' hits
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(FULL, incl, o);
            if (l >= (uint32_t)o) incl += y;
        }
        if (EMIT && hits) {
            const unsigned long long kq = (unsigned long long)w.q << pbits;
            unsigned long long *ks = key + base + count + incl - h;
            uint32_t *vs = val + base + count + incl - h;
            #pragma unroll 1
            for (uint64_t rest = hits; rest; rest &= rest - 1) {
                const uint32_t bit = __ffsll((long long)rest) - 1;
                *ks++ = kq | (uint32_t)(c - (int64_t)A.k + bit);      // p = c - k + bit >= 0; c - k may not be
                *vs++ = v[A.k + bit];
            }
        }
        count += __shfl_sync(FULL, incl, 31);
    }
    if (!EMIT && l == 0) cnt[item] = count;
}

template <bool EMIT>
__global__ void __launch_bounds__(BLK) k_approx_edit(ApproxArgs A, uint32_t *cnt, const unsigned long long *item_off,
                                                     int pbits, unsigned long long *key, uint32_t *val) {
    uint8_t v[EDIT_BAND];
    edit_walk<EMIT, CutPieces>(A, v, cnt, item_off, pbits, key, val);
}

}  // namespace b200sa
