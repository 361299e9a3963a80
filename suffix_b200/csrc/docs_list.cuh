// docs_list.cuh -- document listing over G (SURVEY 8f-8): which documents contain a query and how often,
// from the range [s, e) of G that k_positions<DocsEnd> finds (Muthukrishnan's array).
//
//   byd   the ranks sorted stably by (doc(G[r]), r): the document sort of docs_tree.cuh; document d's
//         ranks are byd[doc_starts[d], doc_starts[d+1]) in increasing order
//   prev  prev[r] = r' + 1 for the previous rank r' of r's document, 0 for its first rank
//   list  the ranks i in [s, e) with prev[i] <= s: the first rank of each document inside the range
//   tf    lower_bound(d's run of byd, e) - lower_bound(d's run, i) for listed rank i of document d
//
// A query's range is cut into chunks that are level-2 blocks (1024 ranks) of the ansv_levels minima over
// prev, and one warp walks one (query, chunk) item: skip the chunk when its minimum is above s, else
// ballot the 32 level-1 minima <= s, and for each hit block ballot its 32 prev values <= s.  The items of
// a query are independent, so one range over most of G spreads over as many warps as it has chunks.
#pragma once
#include "docs.cuh"

namespace b200sa {

constexpr uint32_t DLIST_CHUNK = 1024;       // ranks per item: one level-2 block
constexpr uint32_t DLIST_BAD_RANGE = 1;      // check bit: a range with s > e or e > n

// Item k of the ranks sorted by document (dk = documents, rk = ranks) is byd[k]; its predecessor in
// the same document gives prev.
__global__ void __launch_bounds__(BLK) k_dlist_prev(const uint32_t *__restrict__ dk, const uint32_t *__restrict__ rk,
                                                    uint32_t n, uint32_t *byd, uint32_t *prev) {
    uint32_t k = blockIdx.x * BLK + threadIdx.x;
    if (k >= n) return;
    uint32_t r = rk[k];
    byd[k] = r;
    prev[r] = (k > 0 && dk[k - 1] == dk[k]) ? rk[k - 1] + 1 : 0u;
}

// Scan input over queries 0..nq (entry nq is 0): the number of chunks of [s, e); a bad range counts 0
// and sets the check bit.
struct DListChunks {
    const uint32_t *qs, *qe;
    uint32_t nq, n;
    uint32_t *flag;
    __device__ unsigned long long operator()(uint64_t q) const {
        if (q >= nq) return 0ull;
        uint32_t s = qs[q], e = qe[q];
        if (s > e || e > n) {
            atomicOr(flag, DLIST_BAD_RANGE);
            return 0ull;
        }
        return s < e ? (unsigned long long)((e - 1) / DLIST_CHUNK - s / DLIST_CHUNK + 1) : 0ull;
    }
};
struct InCount64 {                           // u32 counts of `items` entries, 0 past them
    const uint32_t *a;
    uint64_t items;
    __device__ unsigned long long operator()(uint64_t i) const { return i < items ? a[i] : 0u; }
};
struct OutStoreExcl64 {
    unsigned long long *out;
    __device__ void operator()(uint64_t i, unsigned long long exc, unsigned long long) const { out[i] = exc; }
};

// Item `item` of the ranges [rs[r], re[r]) cut into chunks, item_start[r] being range r's first item: its range
// r (the last one whose first item <= item), its chunk blk of DLIST_CHUNK ranks and the ranks [lo, hi) of the
// range inside that chunk.
struct DListItem {
    uint32_t r;
    uint64_t blk, lo, hi;
};
__device__ __forceinline__ DListItem dlist_item(const unsigned long long *item_start, uint32_t nr, const uint32_t *rs,
                                                const uint32_t *re, uint64_t item) {
    uint32_t a = 0, b = nr;
    while (b - a > 1) {
        const uint32_t mid = a + (b - a) / 2;
        if (item_start[mid] <= item) a = mid; else b = mid;
    }
    const uint32_t s = rs[a], e = re[a];
    const uint64_t blk = s / DLIST_CHUNK + (item - item_start[a]);
    const uint64_t lo = blk * DLIST_CHUNK > s ? blk * DLIST_CHUNK : s;
    const uint64_t hi = blk * DLIST_CHUNK + DLIST_CHUNK < e ? blk * DLIST_CHUNK + DLIST_CHUNK : e;
    return {a, blk, lo, hi};
}

struct DListArgs {
    AnsvLevels L;                            // lv[0] = prev; lv[1] / lv[2] exist when n > 32 / n > 1024
    const uint32_t *qs, *qe;
    const unsigned long long *item_start;    // [nq + 1]: first item of each query (exclusive scan of chunks)
    uint32_t nq;
    uint64_t items;
};

// EMIT = false: cnt[item] = the listed ranks of the item.  EMIT = true: the same walk writes, from
// item_off[item] on and in rank order, the document of each listed rank and (tf non-null) its count.
template <bool EMIT>
__global__ void __launch_bounds__(BLK) k_dlist(DListArgs A, uint32_t *cnt, const unsigned long long *item_off,
                                               const uint32_t *__restrict__ g, const uint32_t *__restrict__ starts,
                                               uint32_t ndocs, uint32_t n, const uint32_t *__restrict__ byd,
                                               uint32_t *docs, uint32_t *tf) {
    const uint64_t item = ((uint64_t)blockIdx.x * BLK + threadIdx.x) >> 5;
    if (item >= A.items) return;                                  // whole warps
    const uint32_t l = lane_id();
    const DListItem it = dlist_item(A.item_start, A.nq, A.qs, A.qe, item);
    const uint32_t s = A.qs[it.r], e = A.qe[it.r];
    const uint64_t blk2 = it.blk, lo = it.lo, hi = it.hi;
    uint32_t count = 0;
    const uint64_t base = EMIT ? item_off[item] : 0;
    if (A.L.nlev < 3 || A.L.lv[2][blk2] <= s) {
        const uint64_t b1 = blk2 * 32 + l;                        // lane l: level-1 block b1
        const bool in = b1 * 32 < hi && b1 * 32 + 32 > lo;
        uint32_t m1 = __ballot_sync(FULL, in && (A.L.nlev < 2 || A.L.lv[1][b1] <= s));
        while (m1) {
            const uint32_t k = __ffs(m1) - 1;
            m1 &= m1 - 1;
            const uint64_t i = (blk2 * 32 + k) * 32 + l;
            const bool hit = i >= lo && i < hi && A.L.lv[0][i] <= s;
            const uint32_t m0 = __ballot_sync(FULL, hit);
            if (EMIT && hit) {
                const uint64_t slot = base + count + __popc(m0 & lanemask_lt());
                const uint32_t d = docs_find(starts, ndocs, g[i]);
                docs[slot] = d;
                if (tf) {
                    // lower bounds of i (its own place) and of e in d's run, in lockstep so that the two
                    // loads of a step are in flight together; the run holds i, so it is not empty
                    uint32_t b1 = __ldg(starts + d), b2 = b1, len = docs_end(starts, ndocs, n, d) - b1;
                    while (len > 1) {
                        const uint32_t h = len / 2;
                        const uint32_t v1 = byd[b1 + h], v2 = byd[b2 + h];
                        if (v1 < i) b1 += h;
                        if (v2 < e) b2 += h;
                        len -= h;
                    }
                    b1 += byd[b1] < i;
                    b2 += byd[b2] < e;
                    tf[slot] = b2 - b1;
                }
            }
            count += __popc(m0);
        }
    }
    if (!EMIT && l == 0) cnt[item] = count;
}

// offsets[q] = the output offset of query q's first item, its ranges being q*stride .. q*stride + stride - 1: one
// per query for the listing, the P slots of its pieces for approx.cuh (item_start[nq * stride] = items,
// item_off[items] = total)
__global__ void __launch_bounds__(BLK) k_dlist_qoff(const unsigned long long *__restrict__ item_start,
                                                    const unsigned long long *__restrict__ item_off, uint32_t nq,
                                                    uint32_t stride, unsigned long long *offsets) {
    uint64_t q = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (q > nq) return;
    offsets[q] = item_off[item_start[q * stride]];
}

}  // namespace b200sa
