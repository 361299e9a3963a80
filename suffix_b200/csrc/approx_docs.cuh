// approx_docs.cuh -- the documents that contain each query within k (DESIGN 6b f-19), the B200SA_APPROX_DOCUMENTS
// flag of b200sa_docs_approx_positions_dev.
//
// The call builds q's final list as it would without the flag, but into staging: positions by ascending p (or by
// (p, strand)), so each document's hits are contiguous within a query.  k_adocs_mark marks the hits that start a
// (query, document) segment, one scan of the marks numbers the segments, and k_adocs_offsets reads the caller's
// offsets off that scan at each query's first hit.  When the listing fits, k_adocs_emit writes each segment's
// document at its start and takes the least (d << 1) | minus of the segment with an atomicMin, which does not
// depend on the order of the hits, and k_adocs_dist turns those words into distances.
#pragma once
#include "docs.cuh"

namespace b200sa {

// mark[i] = 1 iff staged hit i is the first of its query's list or its document differs from hit i - 1's.  hoff
// holds the nq + 1 offsets of the staged lists, hpos the htotal positions.
__global__ void __launch_bounds__(BLK) k_adocs_mark(const uint32_t *__restrict__ hpos, uint64_t htotal,
                                                    const unsigned long long *__restrict__ hoff, uint32_t nq,
                                                    const uint32_t *__restrict__ starts, uint32_t ndocs,
                                                    uint32_t *mark) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= htotal) return;
    uint32_t a = 0, b = nq;                                       // the query of hit i: the last q with hoff[q] <= i
    while (b - a > 1) {
        const uint32_t mid = a + (b - a) / 2;
        if (hoff[mid] <= i) a = mid; else b = mid;
    }
    mark[i] = hoff[a] == i || docs_find(starts, ndocs, hpos[i]) != docs_find(starts, ndocs, hpos[i - 1]);
}

// offsets[q] = seg[hoff[q]] for q <= nq: the segments before q's first hit (seg is the exclusive scan of the
// marks, htotal + 1 entries).
__global__ void __launch_bounds__(BLK) k_adocs_offsets(const unsigned long long *__restrict__ hoff,
                                                       const unsigned long long *__restrict__ seg, uint32_t nq,
                                                       unsigned long long *offsets) {
    const uint64_t q = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (q <= nq) offsets[q] = seg[hoff[q]];
}

// Hit i lies in segment seg[i + 1] - 1 and starts it when seg[i + 1] > seg[i]: the start writes the document to
// docs; every hit folds (d << 1) | minus of its distance into least[segment] (pre-set to ~0) when least is set.
__global__ void __launch_bounds__(BLK) k_adocs_emit(const uint32_t *__restrict__ hpos,
                                                    const uint32_t *__restrict__ hmis, uint64_t htotal,
                                                    const unsigned long long *__restrict__ seg,
                                                    const uint32_t *__restrict__ starts, uint32_t ndocs,
                                                    uint32_t *docs, uint32_t *least) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= htotal) return;
    const uint64_t lo = seg[i], hi = seg[i + 1];
    if (hi != lo) docs[lo] = docs_find(starts, ndocs, hpos[i]);
    if (least) {
        const uint32_t v = hmis[i];
        atomicMin(least + hi - 1, (v & ~B200SA_APPROX_MINUS) << 1 | v >> 31);
    }
}

// dist[j] = the least distance of listed document j, with B200SA_APPROX_MINUS when its first hit in (d, strand)
// order is a minus hit.
__global__ void __launch_bounds__(BLK) k_adocs_dist(const uint32_t *__restrict__ least, uint64_t total,
                                                    uint32_t *dist) {
    const uint64_t j = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (j >= total) return;
    const uint32_t w = least[j];
    dist[j] = w >> 1 | (w & 1u ? B200SA_APPROX_MINUS : 0u);
}

}  // namespace b200sa
