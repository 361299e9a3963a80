// best.cuh -- the best approximate occurrences of each query (DESIGN 6b f-16), the B200SA_APPROX_BEST flag of
// the approximate-positions entry points.
//
// Rounds t = 0, 1, ..., threshold each search the live queries at threshold t with the kernels of approx.cuh
// and edit.cuh, on a compacted batch: a scan over the queries picks the live ones, and k_best_gather copies
// their bytes into one buffer with a rebased q_off.  best[q] is the first round that counted an occurrence for q
// (BEST_NONE before), so best(q) = best[q]: round t finds every p with d(p) <= t.  q is live in round t while
// best[q] = BEST_NONE or t <= best[q] + s, and its count is its count in its last live round, the round
// t(q) = min(threshold, best(q) + s).  Emission then runs once per distinct t(q), over the queries that end
// there, and k_best_scatter moves each group's sorted (q, p) keys to the query's place in the caller's arrays.
#pragma once
#include "approx.cuh"

namespace b200sa {

constexpr uint8_t BEST_NONE = 0xFF;

// Scan input over queries 0..nq (entry nq is 0): (1 << 32) | m for a picked query, else 0.  Its exclusive sum is
// (index in the batch << 32) | byte offset in the batch: the bytes sum below 2^32 (q_bytes <= B200SA_MAX_N), so
// nothing carries.  Live (group = false): m > 0 and t <= best + s or no best yet; group: t(q) = t.
struct BestPick {
    const uint64_t *qoff;
    const uint8_t *best;
    uint32_t nq, t, s, k;
    bool group;
    __device__ unsigned long long operator()(uint64_t q) const {
        if (q >= nq) return 0ull;
        const uint32_t m = (uint32_t)(qoff[q + 1] - qoff[q]), b = best[q];
        const bool in = group ? b != BEST_NONE && min(k, b + s) == t
                              : m > 0 && (b == BEST_NONE || t <= b + s);
        return in ? (1ull << 32) | m : 0ull;
    }
};
// map[i] = the query of batch entry i, coff[i] = its byte offset in the batch, coff[batch size] = the bytes.
struct BestPickOut {
    uint32_t nq;
    uint32_t *map;
    uint64_t *coff;
    __device__ void operator()(uint64_t q, unsigned long long exc, unsigned long long v) const {
        if (v || q == nq) coff[exc >> 32] = (uint32_t)exc;
        if (v) map[exc >> 32] = (uint32_t)q;
    }
};

// The batch's query bytes: one warp per batch entry.
__global__ void __launch_bounds__(BLK) k_best_gather(const uint8_t *__restrict__ qs, const uint64_t *__restrict__ qoff,
                                                     const uint32_t *__restrict__ map, const uint64_t *__restrict__ coff,
                                                     uint32_t nb, uint8_t *out) {
    const uint64_t i = ((uint64_t)blockIdx.x * BLK + threadIdx.x) >> 5;
    if (i >= nb) return;
    const uint8_t *src = qs + qoff[map[i]];
    const uint64_t o = coff[i], m = coff[i + 1] - o;
    for (uint64_t x = lane_id(); x < m; x += 32) out[o + x] = src[x];
}

// After round t's count: cnt and best of each batch entry's query from the round's offsets, and bit t of *ended
// when a query with an occurrence has its last live round here.
__global__ void __launch_bounds__(BLK) k_best_update(const uint32_t *__restrict__ map,
                                                     const unsigned long long *__restrict__ roff, uint32_t nb,
                                                     uint32_t t, uint32_t s, uint32_t k, uint8_t *best, uint32_t *cnt,
                                                     uint32_t *ended) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= nb) return;
    const uint32_t q = map[i], c = (uint32_t)(roff[i + 1] - roff[i]);
    uint32_t b = best[q];
    cnt[q] = c;
    if (b == BEST_NONE && c > 0) best[q] = (uint8_t)(b = t);
    if (b != BEST_NONE && (t == k || t == b + s)) atomicOr(ended, 1u << t);
}

// One group's sorted keys (batch entry << pbits) | p and values into the caller's arrays at the query's offset
// (mis may be NULL); goff = the group's own offsets.
__global__ void __launch_bounds__(BLK) k_best_scatter(const unsigned long long *__restrict__ key,
                                                      const uint32_t *__restrict__ val, uint64_t total, int pbits,
                                                      const unsigned long long *__restrict__ goff,
                                                      const uint32_t *__restrict__ map,
                                                      const unsigned long long *__restrict__ offsets, uint32_t *pos,
                                                      uint32_t *mis) {
    const uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= total) return;
    const unsigned long long kk = key[i];
    const uint32_t e = (uint32_t)(kk >> pbits);
    const uint64_t dst = offsets[map[e]] + (i - goff[e]);
    pos[dst] = (uint32_t)(kk & ((1ull << pbits) - 1));
    if (mis) mis[dst] = val[i];
}

}  // namespace b200sa
