// bulge.cuh -- separate budgets for substitutions, DNA bulges and RNA bulges under the edit metric (DESIGN 6b
// f-22), the B200SA_APPROX_BULGES flag of b200sa_docs_approx_positions_dev.
//
// Budgets: t substitutions (X), d DNA bulges (D, a text byte with no query byte) and r RNA bulges (I, a query byte
// with no text byte), d, r <= 3.  p is an occurrence when some alignment of q to T[p, e), e <= end(p), has #X <= t,
// #D <= d and #I <= r; dist(p) is the least #X + #I + #D over those alignments.
// Filter: such an alignment has at most t + d + r edits, so with P = t + d + r + 1 pieces one piece is matched
// exactly (the partition lemma), and the slots, chunks and count -> scan -> emit -> sort flow of approx.cuh carry
// over with ApproxArgs::k = t + d + r.  Piece j sits in the text shifted by (#D - #I) before it, in [-r, d]: a
// candidate s of piece j (c = s - o_j) considers the starts p in [c - d, c + r], at most 7.
// Verification: the layered reversed Sellers DP.  F(x, t, i, e) is the least #X of an alignment of q[x, m) to a
// prefix of T[t, de) with at most i I and at most e D moves, saturated at t + 1: a diagonal move adds the miss, I
// and D move to layer (i - 1, e) and (i, e - 1) and add nothing.  Paths from the window's starts stay on the
// 2(d + r) + 1 diagonals [c - d - r, c + d + r], so one DP over that band gives F(0, p, r, d) for all of them;
// p is an occurrence iff F(0, p, r, d) <= t, and dist(p) = min over (i, e) with F(0, p, i, e) <= t of
// F(0, p, i, e) + i + e.  The (r + 1)(d + 1) <= 16 layers of the <= 13 cells of a row sit in shared memory, one
// byte per (cell, layer) and lane, lanes interleaved.
// Reporter: R(p) is the least (i, s'') with piece i exactly at s'' inside p's document and s'' - o_i - p in [-r, d];
// every occurrence has one, and the candidate emits p iff R(p) is itself, so the count pass is exact.  A query
// whose pieces do not fit (m <= t + d + r for CutPieces, the whole-table slot of IupacPieces) keeps the whole-table
// slot, where each rank s reports p = s alone.
// Pieces::FIXED (DESIGN 6b f-21): a fixed q[x] is never X or I, and no D at (x, t) when q[x] or q[x - 1] is fixed.
#pragma once
#include "iupac.cuh"

namespace b200sa {

constexpr uint32_t BULGE_MAX = 3;                                             // d, r <= 3
constexpr int BULGE_CELLS = (BULGE_MAX + 1) * (BULGE_MAX + 1) * (4 * BULGE_MAX + 1);   // layers x band cells
constexpr int BULGE_WARPS = 4;                                                // 26 KB of shared memory per block
constexpr int BULGE_BLK = BULGE_WARPS * 32;

// The search's arguments with the three budgets; A.k = t + d + r and A.P = A.k + 1.
struct BulgeArgs : ApproxArgs {
    uint32_t t, d, r;
};

// Whether candidate (j, s) is R(p) for the start p of [ds, de).  Inline: out of line, the call keeps A and w in
// local memory and the walk spills.
template <class Pieces>
__device__ __forceinline__ bool bulge_reports(const BulgeArgs &A, int64_t p, uint32_t s, const ApproxItem &w,
                                           uint32_t ds, uint32_t de) {
    const int32_t r = (int32_t)A.r, d = (int32_t)A.d;
    for (uint32_t i = 0; i < w.j; i++) {
        const uint2 pi = Pieces::piece(A, w.q, w.m, i);
        for (int32_t e = -r; e <= d; e++)
            if (edit_piece_at(A.text, p + pi.x + e, w.qq + pi.x, pi.y, ds, de)) return false;
    }
    const uint2 pj = Pieces::piece(A, w.q, w.m, w.j);
    for (int64_t x = p + pj.x - r; x < (int64_t)s; x++)
        if (edit_piece_at(A.text, x, w.qq + pj.x, pj.y, ds, de)) return false;
    return true;
}

// dist of row-0 cell b (sv as bulge_verify left it), or t + 1 when no layer is within t
__device__ __forceinline__ uint32_t bulge_dist(const BulgeArgs &A, const uint8_t *sv, uint32_t b) {
    const uint32_t NL = (A.r + 1) * (A.d + 1);
    uint32_t best = 0xFFu;
    for (uint32_t i = 0; i <= A.r; i++)
        for (uint32_t e = 0; e <= A.d; e++) {
            const uint32_t f = sv[(b * NL + i * (A.d + 1) + e) * 32];
            if (f <= A.t) best = min(best, f + i + e);
        }
    return best;
}

// The starts this candidate reports, bit b for p = c - d + b, with *c_out = c.  sv: the lane's cells, cell
// (b, layer) at sv[(b * NL + layer) * 32], left holding row 0 for bulge_dist (cell b + r of p = c - d + b).
template <class Pieces>
__device__ __forceinline__ uint32_t bulge_verify(const BulgeArgs &A, const ApproxItem &w, uint32_t s, uint8_t *sv,
                                                 int64_t *c_out) {
    const uint32_t d = A.d, r = A.r, NL = (r + 1) * (d + 1), D1 = d + 1;
    const int32_t W = 2 * (int32_t)(d + r) + 1;
    const uint32_t INF = A.t + 1;
    const uint8_t *__restrict__ qq = w.qq;
    const uint32_t m = w.m;
    uint32_t ds, de;
    approx_doc(A, s, &ds, &de);
    const int64_t c = (int64_t)s - w.oj, base = c - (int64_t)(d + r);
    *c_out = c;
    for (int32_t b = 0; b < W; b++) {                      // row m: the empty rest of the query ends anywhere
        const int64_t t = base + m + b;
        const uint8_t y = (t >= (int64_t)ds && t <= (int64_t)de) ? 0 : (uint8_t)INF;
        for (uint32_t L = 0; L < NL; L++) sv[(b * NL + L) * 32] = y;
    }
    for (int64_t x = (int64_t)m - 1; x >= 0; x--) {        // in place, b downwards: cell b - 1 is still row x + 1
        const uint32_t qc = __ldg(qq + x);
        bool fx = false, nodel = false;                    // q[x] is fixed; the row has no D move
        if constexpr (Pieces::FIXED) {
            const uint8_t *__restrict__ mk = Pieces::marks(A, qq);
            fx = __ldg(mk + x) != 0;
            nodel = fx || (x > 0 && __ldg(mk + x - 1) != 0);
        }
        uint32_t low = INF;
        for (int32_t b = W - 1; b >= 0; b--) {
            const int64_t t = base + x + b;
            const bool txt = t >= (int64_t)ds && t < (int64_t)de;
            uint32_t mi = 1;
            if (txt) {
                if constexpr (Pieces::CLASSES) mi = Pieces::miss(__ldg(A.text + t), qc);
                else mi = __ldg(A.text + t) != qc;
            }
            const bool diag = txt && !(fx && mi);
            const bool ins = (txt || t == (int64_t)de) && !fx && b > 0;   // the row below, one cell down
            const bool del = txt && !nodel && b + 1 < W;                  // this row, one cell up
            uint8_t *cell = sv + (uint32_t)b * NL * 32;
            const uint8_t *down = ins ? cell - NL * 32 : cell, *up = del ? cell + NL * 32 : cell;   // cells b -/+ 1
            for (uint32_t L = 0; L < NL; L++) {
                const uint32_t i = L / D1, e = L - i * D1;
                uint32_t y = diag ? cell[L * 32] + mi : INF;
                if (ins && i > 0) y = min(y, (uint32_t)down[(L - D1) * 32]);
                if (del && e > 0) y = min(y, (uint32_t)up[(L - 1) * 32]);
                y = min(y, INF);
                cell[L * 32] = (uint8_t)y;
                low = min(low, y);
            }
        }
        if (low > A.t) return 0;                           // every path to row 0 passes this row
    }
    const uint32_t full = NL - 1;                          // layer (r, d)
    if (w.whole) return sv[((d + r) * NL + full) * 32] <= A.t ? 1u << d : 0u;
    const int64_t lo = max((int64_t)ds, c - (int64_t)d), hi = min((int64_t)de - 1, c + (int64_t)r);
    uint32_t hits = 0;
    for (int64_t p = lo; p <= hi; p++) {
        const uint32_t b = (uint32_t)(p - (c - (int64_t)d));
        if (sv[((b + r) * NL + full) * 32] <= A.t && bulge_reports<Pieces>(A, p, s, w, ds, de)) hits |= 1u << b;
    }
    return hits;
}

// EMIT = false: cnt[item] = the occurrences the item reports.  EMIT = true: the same walk writes them from
// item_off[item] on: key = (q << pbits) | p, val = dist(p).  One warp per item, BULGE_BLK threads per block.
template <bool EMIT, class Pieces>
__global__ void __launch_bounds__(BULGE_BLK) k_approx_bulge(BulgeArgs A, uint32_t *cnt,
                                                            const unsigned long long *item_off, int pbits,
                                                            unsigned long long *key, uint32_t *val) {
    __shared__ uint8_t s_cells[BULGE_WARPS * BULGE_CELLS * 32];
    const uint64_t item = ((uint64_t)blockIdx.x * BULGE_BLK + threadIdx.x) >> 5;
    if (item >= A.items) return;                                  // whole warps
    const uint32_t l = lane_id();
    uint8_t *sv = s_cells + (threadIdx.x >> 5) * BULGE_CELLS * 32 + l;
    const ApproxItem w = approx_item<Pieces>(A, item);
    const uint64_t base = EMIT ? item_off[item] : 0;
    uint32_t count = 0;
    for (uint64_t i0 = w.lo; i0 < w.hi; i0 += 32) {               // the same trip count on every lane
        const uint64_t i = i0 + l;
        int64_t c = 0;
        const uint32_t hits = i < w.hi ? bulge_verify<Pieces>(A, w, A.sa[i], sv, &c) : 0;
        const uint32_t h = __popc(hits);
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
            for (uint32_t rest = hits; rest; rest &= rest - 1) {
                const uint32_t bit = __ffs(rest) - 1;
                *ks++ = kq | (uint32_t)(c - (int64_t)A.d + bit);  // p = c - d + bit >= 0; c - d may not be
                *vs++ = bulge_dist(A, sv, bit + A.r);
            }
        }
        count += __shfl_sync(FULL, incl, 31);
    }
    if (!EMIT && l == 0) cnt[item] = count;
}

}  // namespace b200sa
