// align.cuh -- the alignment of every approximate occurrence as CIGAR operations (DESIGN 6b f-20), the
// B200SA_APPROX_ALIGN flag of b200sa_docs_approx_positions_dev.
//
// The call builds q's final list as it would without the flag, but into the staging of approx_docs.cuh.  A count
// kernel aligns every staged hit and keeps its operations, merged into BAM words (len << 4 | code), at a fixed
// stride of 2k + 1 words per hit (a hit at distance d has at most 2d + 1 operations); a scan of the counts gives
// each hit's first entry, k_adocs_offsets reads the caller's offsets off it, and k_align_emit copies the words.
//
// Hamming (k_align_hamming, one thread per hit): position x of the window is = or X.
// Edit (k_align_edit, one warp per hit): D(x, t) is the least cost of aligning Q[x, m) to a prefix of T[t, E),
// E the end of p's document; rows x = m - 1 .. 0 are computed over the 2d + 1 diagonals t - p - x in [-d, d]
// with values saturated at d + 1.  Lane l holds diagonals l and l + 32.  The diagonal move and the insertion come
// from the row below (same diagonal, one diagonal down), the deletion D(x, t + 1) + 1 is a suffix minimum of
// D + diagonal over the row, taken with shuffles.  Each row's 2-bit move choices (4 ballots, 16 bytes) go to
// shared memory; lane 0 then walks them forward from (0, p).  Every cell of the canonical walk lies in the band,
// and a neighbour that is on an optimal continuation has an in-band optimal path, so the banded choices are the
// full DP's.  D(0, p) must equal the staged d; a difference sets the error word (never expected).
// B200SA_APPROX_FIXED (DESIGN 6b f-21): the Hamming words need nothing new (a fixed position of a hit always
// matches); k_align_edit<true> keeps X and I off fixed symbols and has no D in a row x where Q[x] or Q[x - 1] is
// fixed, in its DP and in its move choices, so the walk takes the first allowed move.
#pragma once
#include "bulge.cuh"
#include "strand.cuh"

namespace b200sa {

enum : uint32_t { ALIGN_I = 1, ALIGN_D = 2, ALIGN_EQ = 7, ALIGN_X = 8 };

// The staged hits and what aligning them reads.  qs: the queries (the canonical copy with iupac), hoff the
// nq + 1 offsets of the staged lists, hpos / hmis the htotal positions and distances (B200SA_APPROX_MINUS on a
// minus hit); ops gets stride words per hit, cnt the number used, err is set on a broken invariant.
struct AlignArgs {
    const uint8_t *text;
    const uint32_t *starts;
    uint32_t ndocs, n;
    const uint8_t *qs;
    const uint64_t *qoff;
    uint32_t nq;
    uint32_t fixed;                          // B200SA_APPROX_FIXED: the marks of the query bytes start at qs + fixed
    const unsigned long long *hoff;
    const uint32_t *hpos, *hmis;
    uint64_t htotal;
    bool iupac;
    uint32_t stride;
    uint32_t *ops, *cnt, *err;
};

// Query symbol x of hit (o, m, minus): q[x], or rc(q)[x] = comp(q[m - 1 - x]) on a minus hit.
struct AlignQuery {
    const uint8_t *q;
    uint32_t m;
    bool minus, iupac;
    __device__ __forceinline__ uint32_t at(uint32_t x) const {
        return minus ? strand_comp(__ldg(q + m - 1 - x), iupac) : __ldg(q + x);
    }
    __device__ __forceinline__ bool match(uint32_t t, uint32_t c) const { return iupac ? iupac_in(t, c) : t == c; }
};

__device__ __forceinline__ AlignQuery align_query(const AlignArgs &A, uint64_t i) {
    uint32_t a = 0, b = A.nq;                                     // the query of hit i: the last q with hoff[q] <= i
    while (b - a > 1) {
        const uint32_t mid = a + (b - a) / 2;
        if (A.hoff[mid] <= i) a = mid; else b = mid;
    }
    const uint64_t o = A.qoff[a];
    return AlignQuery{A.qs + o, (uint32_t)(A.qoff[a + 1] - o), (A.hmis[i] & B200SA_APPROX_MINUS) != 0, A.iupac};
}

// Merges adjacent moves with one code into BAM words at out[0, stride).
struct AlignSink {
    uint32_t *out, stride, n = 0, code = 0, len = 0;
    __device__ __forceinline__ void flush() {
        if (len && n < stride) out[n] = len << 4 | code;
        if (len) n++;
    }
    __device__ __forceinline__ void push(uint32_t c) {
        if (c == code) { len++; return; }
        flush();
        code = c;
        len = 1;
    }
};

// One thread per staged hit.
__global__ void __launch_bounds__(BLK) k_align_hamming(AlignArgs A) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= A.htotal) return;
    const AlignQuery Q = align_query(A, i);
    const uint8_t *__restrict__ t = A.text + A.hpos[i];
    AlignSink s{A.ops + i * A.stride, A.stride};
    uint32_t x_count = 0;
    for (uint32_t x = 0; x < Q.m; x++) {
        const bool eq = Q.match(__ldg(t + x), Q.at(x));
        x_count += !eq;
        s.push(eq ? ALIGN_EQ : ALIGN_X);
    }
    s.flush();
    A.cnt[i] = s.n;
    if (x_count != (A.hmis[i] & ~B200SA_APPROX_MINUS) || s.n > A.stride) atomicOr(A.err, 1u);
}

// One warp per staged hit; rows words of dynamic shared memory (4 per query row) per warp, rows >= the longest
// query of the batch.  The block has blockDim.x / 32 warps.  FIXED: A.fixed marks the fixed symbols of q.
template <bool FIXED>
__global__ void __launch_bounds__(BLK) k_align_edit(AlignArgs A, uint32_t rows) {
    extern __shared__ uint4 s_moves[];
    const uint32_t l = lane_id(), w = threadIdx.x >> 5;
    const uint64_t i = (uint64_t)blockIdx.x * (blockDim.x >> 5) + w;
    if (i >= A.htotal) return;
    uint4 *mv = s_moves + (size_t)w * rows;
    const AlignQuery Q = align_query(A, i);
    const uint32_t p = A.hpos[i], d = A.hmis[i] & ~B200SA_APPROX_MINUS;
    const uint32_t E = docs_end(A.starts, A.ndocs, A.n, docs_find(A.starts, A.ndocs, p));
    const int32_t INF = (int32_t)d + 1, W = 2 * (int32_t)d + 1, j0 = (int32_t)l, j1 = (int32_t)l + 32;
    const bool wide = W > 32;                                     // uniform: the upper half holds cells
    // cell j of row x is t = p + x + j - d; a cell with t < p or t > E is outside the DP and holds INF
    auto tt = [&](uint32_t x, int32_t j) { return (int64_t)p + x + j - (int32_t)d; };
    auto in = [&](uint32_t x, int32_t j) { const int64_t t = tt(x, j); return j < W && t >= p && t <= E; };
    int32_t r0 = in(Q.m, j0) ? 0 : INF, r1 = in(Q.m, j1) ? 0 : INF;   // row m: D(m, t) = 0
    const uint8_t *__restrict__ mk = Q.q + A.fixed;
    auto fixed = [&](uint32_t x) { return __ldg(mk + (Q.minus ? Q.m - 1 - x : x)) != 0; };   // Q[x] is fixed
    for (uint32_t x = Q.m; x-- > 0;) {
        const uint32_t qc = Q.at(x);
        bool fx = false, nodel = false;                           // Q[x] is fixed; the row has no D move
        if constexpr (FIXED) {
            fx = fixed(x);
            nodel = fx || (x > 0 && fixed(x - 1));
        }
        // the row below at diagonal j - 1 (the insertion's source)
        int32_t u0 = __shfl_up_sync(0xffffffffu, r0, 1), u1 = __shfl_up_sync(0xffffffffu, r1, 1);
        const int32_t top = __shfl_sync(0xffffffffu, r0, 31);
        if (l == 0) { u0 = INF; u1 = top; }
        int32_t a0 = INF, a1 = INF, m0 = 1, m1 = 1;
        const bool v0 = in(x, j0), v1 = in(x, j1);
        const int64_t t0 = tt(x, j0), t1 = tt(x, j1);
        // a fixed Q[x] takes only the diagonal, and only on a match
        if (v0) {
            if (t0 < E) { m0 = !Q.match(__ldg(A.text + t0), qc); a0 = fx && m0 ? INF : r0 + m0; }
            if (!fx) a0 = min(a0, u0 + 1);
        }
        if (v1) {
            if (t1 < E) { m1 = !Q.match(__ldg(A.text + t1), qc); a1 = fx && m1 ? INF : r1 + m1; }
            if (!fx) a1 = min(a1, u1 + 1);
        }
        // the deletion: D(j) = min over j' >= j of a(j') + j' - j, a suffix minimum of a + j (uniform: nodel)
        int32_t s0 = min(a0, INF) + j0, s1 = min(a1, INF) + j1;
        if (!nodel) {
            if (wide) {
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int32_t y = __shfl_down_sync(0xffffffffu, s1, o);
                    if (l + o < 32) s1 = min(s1, y);
                }
            }
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int32_t y = __shfl_down_sync(0xffffffffu, s0, o);
                if (l + o < 32) s0 = min(s0, y);
            }
            if (wide) s0 = min(s0, __shfl_sync(0xffffffffu, s1, 0));
        }
        const int32_t n0 = v0 ? min(s0 - j0, INF) : INF, n1 = v1 ? min(s1 - j1, INF) : INF;
        // the first move that holds and is allowed: 1 diagonal, 2 insertion, 3 deletion
        const uint32_t c0 = (t0 < E && !(fx && m0) && n0 == r0 + m0) ? 1u : !fx && n0 == u0 + 1 ? 2u : 3u;
        const uint32_t c1 = (t1 < E && !(fx && m1) && n1 == r1 + m1) ? 1u : !fx && n1 == u1 + 1 ? 2u : 3u;
        const uint32_t b0 = __ballot_sync(0xffffffffu, c0 & 1u), b1 = __ballot_sync(0xffffffffu, c0 & 2u);
        const uint32_t b2 = __ballot_sync(0xffffffffu, c1 & 1u), b3 = __ballot_sync(0xffffffffu, c1 & 2u);
        if (l == 0) mv[x] = make_uint4(b0, b1, b2, b3);
        r0 = n0;
        r1 = n1;
    }
    const int32_t dist = __shfl_sync(0xffffffffu, (int32_t)d < 32 ? r0 : r1, (int32_t)d & 31);
    __syncwarp();
    if (l != 0) return;
    AlignSink s{A.ops + i * A.stride, A.stride};
    bool bad = dist != (int32_t)d;
    uint32_t x = 0, t = p, cost = 0;
    while (x < Q.m && !bad) {
        const int32_t j = (int32_t)(t - p) - (int32_t)x + (int32_t)d;
        if (j < 0 || j >= W) { bad = true; break; }
        const uint4 r = mv[x];
        const uint32_t lo = j < 32 ? r.x : r.z, hi = j < 32 ? r.y : r.w, b = (uint32_t)j & 31u;
        const uint32_t c = (lo >> b & 1u) | (hi >> b & 1u) << 1;
        if (c == 1u) {
            const bool eq = Q.match(__ldg(A.text + t), Q.at(x));
            cost += !eq;
            s.push(eq ? ALIGN_EQ : ALIGN_X);
            x++;
            t++;
        } else if (c == 2u) {
            cost++;
            s.push(ALIGN_I);
            x++;
        } else {
            cost++;
            s.push(ALIGN_D);
            t++;
        }
    }
    s.flush();
    A.cnt[i] = s.n;
    if (bad || cost != d || t > E || s.n > A.stride) atomicOr(A.err, 1u);
}

// B200SA_APPROX_BULGES (DESIGN 6b f-22): one thread per staged hit i in [h0, h1), budgets tb substitutions, d DNA
// and r RNA bulges.  F(x, t, i, e) of bulge.cuh (the least #X of Q[x, m) against a prefix of T[t, E) with at most i
// I and e D moves, saturated at tb + 1) over the d + r + 1 diagonals t - p - x in [-r, d] of the hit's start, every
// row kept: row x of hit i at scratch + ((i - h0) * rows + x) * (d + r + 1) * NL, cell b = t - p - x + r holding
// its NL = (r + 1)(d + 1) layers.  The walk from (0, p) with budgets (r, d, tb) and cost dist takes the first move,
// diagonal, I, D, after which some layer still meets the budgets within the remaining cost (feasible): the f-20
// order among the moves that keep the hit's cost and budgets.  FIXED: A.fixed marks Q's fixed symbols, whose moves
// are constrained as in k_align_edit<true>.  The minimum of one block per SM lets ptxas keep the walk out of local
// memory (it spills at its default of 48 registers).
template <bool FIXED>
__global__ void __launch_bounds__(BLK, 1) k_align_bulge(AlignArgs A, uint32_t tb, uint32_t d, uint32_t r, uint64_t h0,
                                                     uint64_t h1, uint32_t rows, uint8_t *scratch) {
    const uint64_t i = h0 + (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= h1) return;
    const AlignQuery Q = align_query(A, i);
    const uint32_t p = A.hpos[i], dist = A.hmis[i] & ~B200SA_APPROX_MINUS;
    const uint32_t E = docs_end(A.starts, A.ndocs, A.n, docs_find(A.starts, A.ndocs, p));
    const uint32_t NL = (r + 1) * (d + 1), D1 = d + 1, W = d + r + 1, RB = W * NL, INF = tb + 1;
    uint8_t *F = scratch + (i - h0) * rows * RB;
    const uint8_t *__restrict__ mk = Q.q + A.fixed;
    auto fixed = [&](uint32_t x) { return FIXED && __ldg(mk + (Q.minus ? Q.m - 1 - x : x)) != 0; };
    auto tt = [&](uint32_t x, uint32_t b) { return (int64_t)p + x + b - r; };
    for (uint32_t b = 0; b < W; b++) {                             // row m: D(m, t) = 0
        const int64_t t = tt(Q.m, b);
        const uint8_t y = (t >= p && t <= E) ? 0 : (uint8_t)INF;
        for (uint32_t L = 0; L < NL; L++) F[Q.m * RB + b * NL + L] = y;
    }
    for (uint32_t x = Q.m; x-- > 0;) {
        const uint32_t qc = Q.at(x);
        const bool fx = fixed(x), nodel = fx || (x > 0 && fixed(x - 1));
        uint8_t *cur = F + x * RB;
        const uint8_t *below = cur + RB;
        for (uint32_t b = W; b-- > 0;) {
            const int64_t t = tt(x, b);
            const bool txt = t >= p && t < E;
            const uint32_t mi = txt ? !Q.match(__ldg(A.text + t), qc) : 1u;
            const bool diag = txt && !(fx && mi), ins = (txt || t == E) && !fx && b > 0, del = txt && !nodel && b + 1 < W;
            for (uint32_t L = 0; L < NL; L++) {
                const uint32_t li = L / D1, le = L - li * D1;
                uint32_t y = diag ? below[b * NL + L] + mi : INF;
                if (ins && li > 0) y = min(y, (uint32_t)below[(b - 1) * NL + L - D1]);
                if (del && le > 0) y = min(y, (uint32_t)cur[(b + 1) * NL + L - 1]);
                cur[b * NL + L] = (uint8_t)min(y, INF);
            }
        }
    }
    // some alignment of Q[x, m) to T[t, ..) with <= iu I, <= du D and <= xu X moves costs at most C
    auto feasible = [&](uint32_t x, int64_t t, uint32_t iu, uint32_t du, uint32_t xu, int32_t C) {
        const int64_t b = t - p - x + r;
        if (b < 0 || b >= W || C < 0) return false;
        const uint8_t *cell = F + x * RB + b * NL;
#pragma unroll 1
        for (uint32_t li = 0; li <= iu; li++)
#pragma unroll 1
            for (uint32_t le = 0; le <= du; le++) {
                const uint32_t f = cell[li * D1 + le];
                if (f <= xu && (int32_t)(f + li + le) <= C) return true;
            }
        return false;
    };
    AlignSink s{A.ops + i * A.stride, A.stride};
    // the hit's distance is the least cost within the budgets
    bool bad = !feasible(0, p, r, d, tb, (int32_t)dist) || feasible(0, p, r, d, tb, (int32_t)dist - 1);
    uint32_t x = 0, iu = r, du = d, xu = tb;
    int32_t C = (int32_t)dist;
    int64_t t = p;
    while (x < Q.m && !bad) {
        const bool fx = fixed(x), nodel = fx || (x > 0 && fixed(x - 1));
        if (t < E) {
            const uint32_t mi = !Q.match(__ldg(A.text + t), Q.at(x));
            if (!(fx && mi) && mi <= xu && feasible(x + 1, t + 1, iu, du, xu - mi, C - (int32_t)mi)) {
                s.push(mi ? ALIGN_X : ALIGN_EQ);
                x++;
                t++;
                xu -= mi;
                C -= (int32_t)mi;
                continue;
            }
        }
        if (!fx && iu > 0 && feasible(x + 1, t, iu - 1, du, xu, C - 1)) {
            s.push(ALIGN_I);
            x++;
            iu--;
            C--;
            continue;
        }
        if (!nodel && t < E && du > 0 && feasible(x, t + 1, iu, du - 1, xu, C - 1)) {
            s.push(ALIGN_D);
            t++;
            du--;
            C--;
            continue;
        }
        bad = true;
    }
    s.flush();
    A.cnt[i] = s.n;
    if (bad || C != 0 || s.n > A.stride) atomicOr(A.err, 1u);
}

// Hit i's cnt[i] words at its first entry seg[i]: d_pos gets p, d_mis the word with B200SA_APPROX_MINUS from the
// hit's distance.
__global__ void __launch_bounds__(BLK) k_align_emit(const uint32_t *__restrict__ hpos,
                                                    const uint32_t *__restrict__ hmis, uint64_t htotal,
                                                    const unsigned long long *__restrict__ seg,
                                                    const uint32_t *__restrict__ cnt,
                                                    const uint32_t *__restrict__ ops, uint32_t stride,
                                                    uint32_t *pos, uint32_t *mis) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= htotal) return;
    const uint64_t o = seg[i];
    const uint32_t p = hpos[i], minus = hmis[i] & B200SA_APPROX_MINUS, c = cnt[i];
    for (uint32_t j = 0; j < c; j++) {
        pos[o + j] = p;
        mis[o + j] = ops[i * stride + j] | minus;
    }
}

// *mmax = the longest of the nq queries (atomicMax).
__global__ void __launch_bounds__(BLK) k_align_mmax(const uint64_t *__restrict__ qoff, uint32_t nq, uint32_t *mmax) {
    const uint64_t q = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (q < nq) atomicMax(mmax, (uint32_t)(qoff[q + 1] - qoff[q]));
}

}  // namespace b200sa
