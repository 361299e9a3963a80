// loci.cuh -- one hit per locus (DESIGN 6b f-23), the B200SA_APPROX_LOCI flag of b200sa_docs_approx_positions_dev.
//
// The call stages q's final list as B200SA_APPROX_DOCUMENTS does: by (p, strand), so within a query each strand's
// hits ascend in p and each document's hits are contiguous.  Two max scans run over the staged list with one 32-bit
// channel per strand (+ in the low word, - in the high word), so a chain of any length crosses tiles through the
// scan's look-back, never through a serial loop:
//  - the first carries the last hit index + 1 of each strand: a hit is the head of its locus unless the previous hit
//    of its strand is of its query and document and starts less than m = |q| bytes before it;
//  - the second carries the last head index + 1 of each strand, so every hit learns its head (the locus id) and
//    folds (d << 32) | p into least[head] with an atomicMin, which does not depend on the order of the hits.
// A hit whose key is its locus's least is the representative; a sum scan of those marks places them and gives the
// offsets (k_adocs_offsets), and k_loci_emit copies them.  Hit indices take 32 bits: fewer than 2^32 - 1 hits.
#pragma once
#include "docs.cuh"

namespace b200sa {

// max over each 32-bit half on its own: commutative, as k_scan_lb's reductions require
struct OpMax2x32 {
    using T = unsigned long long;
    __device__ __forceinline__ static T id() { return 0ull; }
    __device__ __forceinline__ static T op(T a, T b) {
        const uint32_t lo = max((uint32_t)a, (uint32_t)b), hi = max((uint32_t)(a >> 32), (uint32_t)(b >> 32));
        return (T)hi << 32 | lo;
    }
};

// The strand's channel of a 2x32 value: the high word for a - hit (B200SA_APPROX_MINUS in its distance).
__device__ __forceinline__ unsigned long long loci_channel(uint32_t mis, unsigned long long v) {
    return v << (mis >> 31 ? 32 : 0);
}
__device__ __forceinline__ uint32_t loci_read(uint32_t mis, unsigned long long v) {
    return (uint32_t)(mis >> 31 ? v >> 32 : v);
}

// The query of staged hit i: the last q with hoff[q] <= i.
__device__ __forceinline__ uint32_t loci_query(const unsigned long long *__restrict__ hoff, uint32_t nq, uint64_t i) {
    uint32_t a = 0, b = nq;
    while (b - a > 1) {
        const uint32_t mid = a + (b - a) / 2;
        if (hoff[mid] <= i) a = mid; else b = mid;
    }
    return a;
}

// First scan: in(i) = i + 1 in i's channel.
struct LociPrevIn {
    const uint32_t *mis;
    __device__ unsigned long long operator()(uint64_t i) const { return loci_channel(mis[i], i + 1); }
};
// mark[i] = 1 iff hit i is a head.  exc's channel is the index + 1 of the previous hit of i's strand (0: none).
struct LociPrevOut {
    const uint32_t *pos, *mis;
    const unsigned long long *hoff, *q_off;
    uint32_t nq;
    const uint32_t *starts;
    uint32_t ndocs;
    uint32_t *mark;
    __device__ void operator()(uint64_t i, unsigned long long exc, unsigned long long) const {
        const uint32_t prev = loci_read(mis[i], exc);
        bool head = true;
        if (prev) {
            const uint64_t j = prev - 1;
            const uint32_t q = loci_query(hoff, nq, i), p = pos[i], pj = pos[j];
            head = j < hoff[q] || (uint64_t)(p - pj) >= q_off[q + 1] - q_off[q] ||
                   docs_find(starts, ndocs, pj) != docs_find(starts, ndocs, p);
        }
        mark[i] = head;
    }
};

// Second scan: in(i) = i + 1 in i's channel when i is a head, else 0.
struct LociHeadIn {
    const uint32_t *mis, *mark;
    __device__ unsigned long long operator()(uint64_t i) const { return mark[i] ? loci_channel(mis[i], i + 1) : 0ull; }
};
// The inclusive channel is i's head + 1: head[i] (in place of mark[i], which the same thread read) and the atomicMin
// of i's key into least[head] (pre-set to ~0).
struct LociHeadOut {
    const uint32_t *pos, *mis;
    uint32_t *head;
    unsigned long long *least;
    __device__ void operator()(uint64_t i, unsigned long long exc, unsigned long long v) const {
        const uint32_t w = mis[i], h = loci_read(w, OpMax2x32::op(exc, v)) - 1;
        head[i] = h;
        atomicMin(least + h, (unsigned long long)(w & ~B200SA_APPROX_MINUS) << 32 | pos[i]);
    }
};

// Third scan (a sum over htotal + 1 entries): 1 for a representative, the hit whose key is its locus's least.
struct LociKeepIn {
    const uint32_t *pos, *mis, *head;
    const unsigned long long *least;
    uint64_t htotal;
    __device__ unsigned long long operator()(uint64_t i) const {
        if (i >= htotal) return 0ull;
        return least[head[i]] == ((unsigned long long)(mis[i] & ~B200SA_APPROX_MINUS) << 32 | pos[i]);
    }
};

// Hit i is kept when keep[i + 1] > keep[i] (keep: the exclusive scan of the marks); it goes to keep[i].
__global__ void __launch_bounds__(BLK) k_loci_emit(const uint32_t *__restrict__ hpos, const uint32_t *__restrict__ hmis,
                                                   uint64_t htotal, const unsigned long long *__restrict__ keep,
                                                   uint32_t *pos, uint32_t *mis) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= htotal) return;
    const uint64_t at = keep[i];
    if (keep[i + 1] == at) return;
    pos[at] = hpos[i];
    if (mis) mis[at] = hmis[i];
}

}  // namespace b200sa
