// iupac.cuh -- queries written in IUPAC nucleotide codes (DESIGN 6b f-17), the B200SA_APPROX_IUPAC flag of the
// approximate-positions entry points.
//
// A query symbol stands for a class of text bytes: A C G T (U = T) for themselves, the degenerate codes R Y S W
// K M B D H V N for two to four of them, either case.  Only the uppercase text bytes A C G T are in any class.
// k_iupac_code writes the canonical copy of the queries, one byte per byte: the uppercase base of a concrete
// symbol (A C G T U), else the class as a mask of bases (A 1, C 2, G 4, T 8), two or more bits, so below 16.
// Pieces come only from the stretches (maximal runs of concrete symbols, lengths L_i): with t the largest length
// with sum floor(L_i / t) >= P = k + 1, stretch i gives c_i = min(floor(L_i / t), pieces still needed) pieces cut
// as approx_cut cuts a query.  They are disjoint and concrete, so each is one exact range of the table, and the
// partition lemma (which needs k + 1 disjoint pieces, not a cover) keeps the reporters of approx.cuh and edit.cuh
// exact: a window within k has one of them intact.  For a concrete query they are f-14's pieces.  A query with
// sum L_i < P keeps the whole-table slot: every rank is a candidate and is verified in full.  The piece of slot
// q*P + j is (offset, length) in entry q*P + j of the piece table; length 0 marks the whole-table slot.  The table
// follows pe in the same buffer (iupac_table), so the walks find it from ApproxArgs and keep no pointer live; with
// B200SA_APPROX_FIXED the pointer to the batch's marks follows the table (iupac_marks) for the same reason.
// IupacPieces gives the walks these pieces and the class test in place of CutPieces.  FixedIupacPieces adds the
// fixed symbols of B200SA_APPROX_FIXED (DESIGN 6b f-21): the lowercase letters of the query, marked 1 in a copy of
// one byte per query byte beside the canonical one (k_iupac_marks).  A window with a fixed miss is no occurrence and
// the free misses are counted; edit_verify keeps X, I and D off them.  The pieces and reporters are IupacPieces':
// every constrained occurrence is an unconstrained one, so one of the k + 1 pieces is still intact.
#pragma once
#include "edit.cuh"

namespace b200sa {

// The canonical symbol of a query byte, 0 if it is not an IUPAC letter.
__device__ __forceinline__ uint32_t iupac_code(uint32_t b) {
    switch (b | 0x20u) {                                  // lowercase; only 'X' and 'x' map to a letter 'x'
    case 'a': return 'A';
    case 'c': return 'C';
    case 'g': return 'G';
    case 't': case 'u': return 'T';
    case 'r': return 1 | 4;
    case 'y': return 2 | 8;
    case 's': return 2 | 4;
    case 'w': return 1 | 8;
    case 'k': return 4 | 8;
    case 'm': return 1 | 2;
    case 'b': return 2 | 4 | 8;
    case 'd': return 1 | 4 | 8;
    case 'h': return 1 | 2 | 8;
    case 'v': return 1 | 2 | 4;
    case 'n': return 15;
    default: return 0;
    }
}

// Whether text byte t is in the class of canonical symbol c
__device__ __forceinline__ bool iupac_in(uint32_t t, uint32_t c) {
    if (c >= 16) return t == c;
    const uint32_t bit = t == 'A' ? 1u : t == 'C' ? 2u : t == 'G' ? 4u : t == 'T' ? 8u : 0u;
    return (bit & c) != 0;
}

// The canonical copy of the query bytes, and *bad = the least (offset << 8) | byte of a byte that is not an IUPAC
// letter (left at ~0 if there is none).  One thread per byte.
__global__ void __launch_bounds__(BLK) k_iupac_code(const uint8_t *__restrict__ qs, uint64_t bytes, uint8_t *out,
                                                    unsigned long long *bad) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= bytes) return;
    const uint32_t b = qs[i], c = iupac_code(b);
    out[i] = (uint8_t)c;
    if (!c) atomicMin(bad, ((unsigned long long)i << 8) | b);
}

// B200SA_APPROX_FIXED: 1 for a fixed (lowercase) query byte, else 0.  Runs after k_iupac_code accepted every byte
// as a letter, so bit 0x20 tells the case.  One thread per byte.
__global__ void __launch_bounds__(BLK) k_iupac_marks(const uint8_t *__restrict__ qs, uint64_t bytes, uint8_t *out) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i < bytes) out[i] = (qs[i] & 0x20u) ? 1 : 0;
}

// sum over the stretches of qq[0, m) of floor(L_i / t), stopping once it reaches P
__device__ __forceinline__ uint32_t iupac_fit(const uint8_t *__restrict__ qq, uint32_t m, uint32_t t, uint32_t P) {
    uint32_t sum = 0, run = 0;
    for (uint32_t x = 0; x < m && sum < P; x++) {
        if (qq[x] >= 16) {
            if (++run == t) { sum++; run = 0; }
        } else {
            run = 0;
        }
    }
    return sum;
}

// The piece table: nslots (offset, length) entries right after pe[0, nslots), 8-byte aligned as ps starts so.
__device__ __forceinline__ const uint2 *iupac_table(const ApproxArgs &A) {
    return reinterpret_cast<const uint2 *>(A.pe + A.nslots);
}

// B200SA_APPROX_FIXED: the marks of the batch's query bytes, marks[i] for qs[i], whose pointer the host writes after
// the piece table.
__device__ __forceinline__ const uint8_t *iupac_marks(const ApproxArgs &A) {
    return *reinterpret_cast<const uint8_t *const *>(iupac_table(A) + A.nslots);
}

// The piece table and the slot ranges of the canonical queries: pieces / ps / pe[q*P + j] (one thread per query;
// n >= 1).  Unused slots get (0, 0) and an empty range.
template <class EndF>
__global__ void __launch_bounds__(BLK) k_iupac_pieces(const uint8_t *__restrict__ text, uint32_t n,
                                                      const uint32_t *__restrict__ sa, const uint8_t *__restrict__ qs,
                                                      const uint64_t *__restrict__ qoff, uint32_t nq, uint32_t P,
                                                      uint32_t *ps, uint32_t *pe, uint2 *pieces, EndF end) {
    const uint64_t q = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (q >= nq) return;
    const uint8_t *__restrict__ qq = qs + qoff[q];
    const uint32_t m = (uint32_t)(qoff[q + 1] - qoff[q]);
    const uint64_t s0 = q * P;
    uint32_t concrete = 0, j = 0;
    for (uint32_t x = 0; x < m; x++) concrete += qq[x] >= 16;
    if (concrete >= P) {
        uint32_t lo = 1, hi = concrete / P;                // fit(1) >= P; fit falls as t grows
        while (lo < hi) {
            const uint32_t mid = lo + (hi - lo + 1) / 2;
            if (iupac_fit(qq, m, mid, P) >= P) lo = mid; else hi = mid - 1;
        }
        for (uint32_t x = 0; x < m && j < P;) {
            if (qq[x] < 16) { x++; continue; }
            uint32_t y = x;
            while (y < m && qq[y] >= 16) y++;
            const uint32_t L = y - x, cnt = min(L / lo, P - j);
            for (uint32_t i = 0; i < cnt; i++, j++) {
                const uint32_t a = x + approx_cut(L, cnt, i), b = x + approx_cut(L, cnt, i + 1);
                uint32_t s = 0, e = 0;
                positions_range(text, n, sa, qq + a, b - a, end, &s, &e);
                pieces[s0 + j] = make_uint2(a, b - a);
                ps[s0 + j] = s;
                pe[s0 + j] = e;
            }
            x = y;
        }
    } else if (m > 0) {
        pieces[s0] = make_uint2(0, 0);
        ps[s0] = 0;
        pe[s0] = n;
        j = 1;
    }
    for (; j < P; j++) {
        pieces[s0 + j] = make_uint2(0, 0);
        ps[s0 + j] = 0;
        pe[s0 + j] = 0;
    }
}

// The pieces of the piece table and the class test: CutPieces' members for the canonical queries.
struct IupacPieces {
    static __device__ __forceinline__ bool whole(const ApproxArgs &A, uint32_t slot, uint32_t) {
        return iupac_table(A)[slot].y == 0;
    }
    static __device__ __forceinline__ uint32_t off(const ApproxArgs &A, uint32_t slot, uint32_t, uint32_t) {
        return iupac_table(A)[slot].x;
    }
    static __device__ __forceinline__ uint2 piece(const ApproxArgs &A, uint32_t q, uint32_t, uint32_t i) {
        return iupac_table(A)[(uint64_t)q * A.P + i];
    }
    // The class test over all m symbols, then the pieces [0, j) of the query's table.
    static __device__ __forceinline__ bool verify(const ApproxArgs &A, const ApproxItem &w, uint32_t s,
                                                  uint32_t *p_out, uint32_t *mis_out) {
        return verify_marked<false>(A, w, s, p_out, mis_out);
    }
    // FIXED: a miss on a fixed symbol rejects the window, and only the free misses count.  The count over all m
    // symbols bounds the free count from above, and a window with a fixed miss is rejected anyway, so the hot loop
    // stays IupacPieces' and only a window within k reads its marks (then it has no fixed miss and mis is free).
    template <bool FIXED>
    static __device__ __forceinline__ bool verify_marked(const ApproxArgs &A, const ApproxItem &w, uint32_t s,
                                                         uint32_t *p_out, uint32_t *mis_out) {
        if (s < w.oj) return false;
        const uint32_t p = s - w.oj;
        uint32_t ds, de;
        approx_doc(A, s, &ds, &de);
        if (p < ds || (uint64_t)p + w.m > de) return false;
        const uint8_t *__restrict__ t = A.text + p;
        const uint8_t *__restrict__ qq = w.qq;
        uint32_t mis = 0;
        for (uint32_t x = 0; x < w.m; x++) {
            mis += !iupac_in(__ldg(t + x), __ldg(qq + x));
            if (mis > A.k) return false;
        }
        if constexpr (FIXED) {
            const uint8_t *__restrict__ mk = iupac_marks(A) + (qq - A.qs);
            if (mis)
                for (uint32_t x = 0; x < w.m; x++)
                    if (__ldg(mk + x) && !iupac_in(__ldg(t + x), __ldg(qq + x))) return false;
        }
        if (!w.whole) {
            const uint2 *__restrict__ pc = iupac_table(A) + (uint64_t)w.q * A.P;
            for (uint32_t i = 0; i < w.j; i++) {
                const uint2 pi = pc[i];
                if (approx_piece_at(t + pi.x, qq + pi.x, pi.y)) return false;     // slot i reports it
            }
        }
        *p_out = p;
        *mis_out = mis;
        return true;
    }
    static constexpr bool CLASSES = true;
    static constexpr bool FIXED = false;
    static __device__ __forceinline__ bool miss(uint32_t t, uint32_t qc) { return !iupac_in(t, qc); }
    // m may exceed k here, so dist(s) = v[2k] is tested
    static __device__ __forceinline__ uint64_t whole_hits(const uint8_t *v, int32_t k) {
        return v[2 * k] <= (uint32_t)k ? 1ull << k : 0ull;
    }
    // CutPieces::reports with the pieces [0, j] of query q's table; out of line for the same reason.
    static __device__ __noinline__ bool reports(const ApproxArgs &A, int64_t p, uint32_t s,
                                                const uint8_t *__restrict__ qq, uint32_t, uint32_t q, uint32_t j,
                                                uint32_t, uint32_t ds, uint32_t de) {
        const int32_t k = (int32_t)A.k;
        const uint2 *__restrict__ pc = iupac_table(A) + (uint64_t)q * A.P;
        for (uint32_t i = 0; i < j; i++) {
            const uint2 pi = pc[i];
            for (int32_t d = -k; d <= k; d++)
                if (edit_piece_at(A.text, p + pi.x + d, qq + pi.x, pi.y, ds, de)) return false;
        }
        const uint2 pj = pc[j];
        for (int64_t x = p + pj.x - k; x < (int64_t)s; x++)
            if (edit_piece_at(A.text, x, qq + pj.x, pj.y, ds, de)) return false;
        return true;
    }
};

// IupacPieces with the marks of iupac_marks: verify rejects a fixed miss, edit_verify constrains its moves.
struct FixedIupacPieces : IupacPieces {
    static __device__ __forceinline__ bool verify(const ApproxArgs &A, const ApproxItem &w, uint32_t s,
                                                  uint32_t *p_out, uint32_t *mis_out) {
        return verify_marked<true>(A, w, s, p_out, mis_out);
    }
    static constexpr bool FIXED = true;
    // the marks of the query at qq
    static __device__ __forceinline__ const uint8_t *marks(const ApproxArgs &A, const uint8_t *qq) {
        return iupac_marks(A) + (qq - A.qs);
    }
};

// The minimum of 4 blocks per SM lets ptxas use up to 64 registers: left to itself it holds the count pass at 32
// and spills.
template <bool EMIT>
__global__ void __launch_bounds__(BLK, 4) k_approx_iupac(ApproxArgs A, uint32_t *cnt, const unsigned long long *item_off,
                                                         int pbits, unsigned long long *key, uint32_t *val) {
    approx_walk<EMIT, IupacPieces>(A, cnt, item_off, pbits, key, val);
}

template <bool EMIT>
__global__ void __launch_bounds__(BLK) k_approx_edit_iupac(ApproxArgs A, uint32_t *cnt,
                                                           const unsigned long long *item_off, int pbits,
                                                           unsigned long long *key, uint32_t *val) {
    uint8_t v[EDIT_BAND];
    edit_walk<EMIT, IupacPieces>(A, v, cnt, item_off, pbits, key, val);
}

// B200SA_APPROX_FIXED: the IUPAC kernels with FixedIupacPieces, under the same launch bounds.
template <bool EMIT>
__global__ void __launch_bounds__(BLK, 4) k_approx_iupac_fixed(ApproxArgs A, uint32_t *cnt,
                                                               const unsigned long long *item_off, int pbits,
                                                               unsigned long long *key, uint32_t *val) {
    approx_walk<EMIT, FixedIupacPieces>(A, cnt, item_off, pbits, key, val);
}

template <bool EMIT>
__global__ void __launch_bounds__(BLK) k_approx_edit_iupac_fixed(ApproxArgs A, uint32_t *cnt,
                                                                 const unsigned long long *item_off, int pbits,
                                                                 unsigned long long *key, uint32_t *val) {
    uint8_t v[EDIT_BAND];
    edit_walk<EMIT, FixedIupacPieces>(A, v, cnt, item_off, pbits, key, val);
}

}  // namespace b200sa
