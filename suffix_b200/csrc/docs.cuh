// docs.cuh -- the generalized suffix array of many documents without separators (SURVEY 8f-6;
// the reference names it as missing, README.md:60-74, TODO:13-18).
//
// C is the concatenation of the documents, p a position of document d, r_p = end_d - p and
// T_p = C[p, p + r_p).  G sorts the positions by (T_p, d); glcp[i] = lcp(T_{G[i-1]}, T_{G[i]}).
// From SA_C and LCP_C of the concatenation:
//   lo_i  first rank whose suffix shares >= r_p bytes with p = SA_C[i]: i itself when
//         LCP_C[i] < r_p (set U, already in order), else the largest j < i with LCP_C[j] < r_p
//         (set A; ansv_left over the block minima with a per-rank threshold)
//   G     the ranks sorted by (lo, r, d): T_p < T_q iff (lo_p, r_p) < (lo_q, r_q), and equal
//         (lo, r) means equal strings, ordered by document.  A is sorted on its own and merged:
//         element k of sorted A goes to slot k + #U[0, lo) + [lo in U and (r, p) of rank lo < its own];
//         U fills the free slots in rank order.
//   glcp  of neighbours a, b (C-ranks x, y): min(r_a, r_b) if lo_a == lo_b (both are prefixes of
//         the suffix at rank lo), else min(r_a, r_b, min LCP_C(lo_a, lo_b]).
#pragma once
#include "pipeline_kernels.cuh"

namespace b200sa {

constexpr uint32_t DOCS_NONE = 0xffffffffu;
// bits of the doc_starts check word (reported through last_error)
constexpr uint32_t DOCS_BAD_FIRST = 1, DOCS_BAD_ORDER = 2, DOCS_BAD_RANGE = 4;

// document of position p: the last d with starts[d] <= p (an empty document shares its start with
// the next one, so p lands in the non-empty one)
__device__ __forceinline__ uint32_t docs_find(const uint32_t *__restrict__ starts, uint32_t ndocs, uint32_t p) {
    uint32_t lo = 0, hi = ndocs;
    while (hi - lo > 1) {
        uint32_t mid = lo + (hi - lo) / 2;
        if (__ldg(starts + mid) <= p) lo = mid; else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ uint32_t docs_end(const uint32_t *__restrict__ starts, uint32_t ndocs, uint32_t n,
                                             uint32_t d) {
    return d + 1 < ndocs ? __ldg(starts + d + 1) : n;
}

// words[0] |= check bits of doc_starts (starts[0] == 0, ascending, every entry <= n);
// words[1] = max(words[1], longest document)
__global__ void __launch_bounds__(BLK) k_docs_check(const uint32_t *__restrict__ starts, uint32_t ndocs, uint32_t n,
                                                    uint32_t *words) {
    uint32_t d = blockIdx.x * BLK + threadIdx.x, bad = 0, len = 0;
    if (d < ndocs) {
        uint32_t s = starts[d], e = d + 1 < ndocs ? starts[d + 1] : n;
        if (d == 0 && s != 0) bad |= DOCS_BAD_FIRST;
        if (s > n) bad |= DOCS_BAD_RANGE;               // an end above n is the next start, flagged by d + 1
        else if (e < s) bad |= DOCS_BAD_ORDER;
        else if (e <= n) len = e - s;
    }
    bad = __reduce_or_sync(FULL, bad);
    len = __reduce_max_sync(FULL, len);
    if (lane_id() == 0) {
        if (bad) atomicOr(words, bad);
        if (len) atomicMax(words + 1, len);
    }
}

// Scan input over ranks: r of rank i (stored), 1 iff i is in A.  Rank 0 is in U (lcp[0] = 0 < r).
struct DocsSplitIn {
    const uint32_t *sa, *lcp, *starts;
    uint32_t ndocs, n;
    uint32_t *rem;
    __device__ uint32_t operator()(uint64_t i) const {
        uint32_t p = sa[i], r = docs_end(starts, ndocs, n, docs_find(starts, ndocs, p)) - p;
        rem[i] = r;
        return lcp[i] >= r ? 1u : 0u;
    }
};
// Scan output: pre[i] = #A before rank i; U ranks in rank order at list[0, |U|), A ranks at list[|U|, n).
struct DocsSplitOut {
    uint32_t *pre, *list;
    uint32_t n;
    __device__ void operator()(uint64_t i, uint32_t exc, uint32_t v) const {
        pre[i] = exc;
        if (v) list[n - 1 - exc] = (uint32_t)i;
        else list[(uint32_t)i - exc] = (uint32_t)i;
    }
};

// Sort key of the A rank alist[k]: (lo << rb | r), followed by db bits of the document when with_doc.
struct DocsKey {
    AnsvLevels L;
    const uint32_t *sa, *rem, *starts, *alist;
    uint32_t ndocs;
    int rb, db;
    bool with_doc;
    __device__ uint64_t operator()(uint64_t k) const {
        uint32_t i = alist[k], r = rem[i];
        uint64_t key = ((uint64_t)ansv_left<true>(L, i, r) << rb) | r;
        if (with_doc) key = (key << db) | docs_find(starts, ndocs, sa[i]);
        return key;
    }
};
// Document of the A rank alist[k] (first pass of the two-stage sort, when (lo, r, d) needs > 64 bits).
struct DocsDocKey {
    const uint32_t *sa, *starts, *alist;
    uint32_t ndocs;
    __device__ uint32_t operator()(uint64_t k) const { return docs_find(starts, ndocs, sa[alist[k]]); }
};

// Element k of sorted A (C-rank val[k], lo = key[k] >> shift) to its slot of G.
__global__ void __launch_bounds__(BLK) k_docs_place(const uint64_t *__restrict__ key, const uint32_t *__restrict__ val,
                                                    uint32_t na, int shift, const uint32_t *__restrict__ sa,
                                                    const uint32_t *__restrict__ lcp, const uint32_t *__restrict__ rem,
                                                    const uint32_t *__restrict__ pre, uint32_t *gr, uint32_t *glo) {
    uint32_t k = blockIdx.x * BLK + threadIdx.x;
    if (k >= na) return;
    uint32_t i = val[k], lo = (uint32_t)(key[k] >> shift), r = rem[i], rl = rem[lo];
    bool u_first = lcp[lo] < rl && (rl < r || (rl == r && sa[lo] < sa[i]));
    uint32_t s = k + (lo - pre[lo]) + (u_first ? 1u : 0u);
    gr[s] = i;
    glo[s] = lo;
}

// Scan over the slots of G: the free ones (glo == NONE) take the U ranks in rank order.
struct DocsFreeIn {
    const uint32_t *glo;
    __device__ uint32_t operator()(uint64_t s) const { return glo[s] == DOCS_NONE ? 1u : 0u; }
};
struct DocsFreeOut {
    const uint32_t *ulist;
    uint32_t *gr, *glo;
    __device__ void operator()(uint64_t s, uint32_t exc, uint32_t v) const {
        if (v) {
            uint32_t j = ulist[exc];
            gr[s] = j;
            glo[s] = j;
        }
    }
};

// min(m, lv[0][a..b]) for a <= b over the 32-ary block minima: the partial blocks at both ends of a
// level, then the whole blocks between them one level up.
__device__ __forceinline__ uint32_t docs_range_min(const AnsvLevels &L, uint64_t a, uint64_t b, uint32_t m) {
    for (int k = 0; m > 0; k++) {
        const uint32_t *lv = L.lv[k];
        if ((a >> 5) == (b >> 5) || k + 1 >= L.nlev) {
            for (uint64_t j = a; j <= b; j++) m = min(m, lv[j]);
            return m;
        }
        for (uint64_t j = a; j <= (a | 31); j++) m = min(m, lv[j]);
        for (uint64_t j = b & ~(uint64_t)31; j <= b; j++) m = min(m, lv[j]);
        uint64_t na = (a >> 5) + 1, nb = b >> 5;     // whole blocks na .. nb - 1 of level k + 1
        if (na >= nb) return m;
        a = na;
        b = nb - 1;
    }
    return m;
}

// Slot s of G: gsa[s] = SA_C[gr[s]], glcp[s] from the neighbour's C-rank and lo.  gr == null: G is
// SA_C (A is empty, lo = rank).
__global__ void __launch_bounds__(BLK) k_docs_out(const uint32_t *__restrict__ gr, const uint32_t *__restrict__ glo,
                                                  uint32_t n, const uint32_t *__restrict__ sa,
                                                  const uint32_t *__restrict__ rem, AnsvLevels L, uint32_t *gsa,
                                                  uint32_t *glcp) {
    uint32_t s = blockIdx.x * BLK + threadIdx.x;
    if (s >= n) return;
    uint32_t x = gr ? gr[s] : s;
    gsa[s] = sa[x];
    if (!glcp) return;
    uint32_t v = 0;
    if (s > 0) {
        uint32_t y = gr ? gr[s - 1] : s - 1;
        uint32_t lx = gr ? glo[s] : s, ly = gr ? glo[s - 1] : s - 1;
        v = min(rem[x], rem[y]);
        if (lx != ly) v = docs_range_min(L, (uint64_t)ly + 1, lx, v);
    }
    glcp[s] = v;
}

// Batched positions over G: k_positions with every suffix cut at its document's end.
struct DocsEnd {
    const uint32_t *starts;
    uint32_t ndocs, n;
    __device__ __forceinline__ uint32_t operator()(uint32_t p) const {
        return docs_end(starts, ndocs, n, docs_find(starts, ndocs, p));
    }
};

}  // namespace b200sa
