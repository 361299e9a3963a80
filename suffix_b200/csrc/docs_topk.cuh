// docs_topk.cuh -- top-k document retrieval (SURVEY 8f-9): per query the min(k, df) documents of its
// listing (docs_list.cuh) with the largest keys, tf descending, then document ascending.
//
// A round's listing is materialised by k_dlist<true> into X: documents at X[0, R), tf at X[R, 2R) (R = the
// buffer's entries per array), query q's entries at [off[q] - e0, off[q+1] - e0).  The selection compares
//   key(d, tf) = (tf << db) | (ndocs - 1 - d),   db = bit_length(ndocs - 1),
// the order of ((u64)tf << 32) | (0xFFFFFFFF - d) in fewer bits.  The documents of a query are distinct, so
// its keys are unique, and every key is > 0 (tf >= 1), so 0 pads below all of them.
//
// Size classes, chosen per query from df = off[q+1] - off[q]:
//   df <= TOPK_WARP   k_topk_warp: one warp per query, one key per lane, a shuffle bitonic sort.
//   df >  TOPK_WARP   k_topk_tile: one block per tile of <= TOPK_TILE keys in shared memory: a radix select
//                     of the k-th key over the 8-bit digits from the highest bit that varies in the tile
//                     (OR ^ AND of its keys), compaction of the survivors, a bitonic sort of them.  A query
//                     of one tile writes its answer.  A larger one runs in levels: tile t of level i keeps
//                     its min(k, len) best keys, unsorted, at seg + t * k of the other key buffer, so level
//                     i + 1 sees (tiles - 1) * k + min(k, last tile) candidates of the query, until one
//                     tile remains.  Each level reads at most k / TOPK_TILE of the keys of the one before.
// The tiles of a level are numbered by a scan of topk_tiles over the round's queries (0 for the queries of
// the warp class and for those already answered), and a grid-stride loop of blocks walks them.
#pragma once
#include "docs_list.cuh"

namespace b200sa {

constexpr uint32_t TOPK_WARP = 32;          // largest df of the warp class
constexpr uint32_t TOPK_TILE = 4096;        // keys per tile of the block class (32 KB of shared memory)
constexpr uint32_t TOPK_KMAX = 1024;        // B200SA_TOPK_MAX

struct TopkArgs {
    const unsigned long long *off;          // [nq + 1] listing offsets of the whole batch
    uint64_t e0;                            // the round's first entry: off[q0]
    uint64_t R;                             // X holds documents at [0, R), tf at [R, 2R)
    uint32_t q0, nqr;                       // the round's queries [q0, q0 + nqr)
    uint32_t k, ndocs, db;
    uint32_t *docs, *tf;                    // outputs, k slots per query
};

__device__ __forceinline__ unsigned long long topk_key(const TopkArgs &P, uint32_t d, uint32_t tf) {
    return ((unsigned long long)tf << P.db) | (P.ndocs - 1 - d);
}
__device__ __forceinline__ void topk_put(const TopkArgs &P, uint64_t slot, unsigned long long key) {
    P.tf[slot] = (uint32_t)(key >> P.db);
    P.docs[slot] = P.ndocs - 1 - (uint32_t)(key & ((1ull << P.db) - 1));
}

// Tiles of a query with df entries at `level` (0 when it is of the warp class or answered at an earlier
// level); *len = its candidates at that level.  The host mirrors this recurrence to count the levels.
__device__ __forceinline__ uint32_t topk_tiles(uint64_t df, uint32_t k, uint32_t level, uint64_t *len) {
    if (df <= TOPK_WARP) return 0;
    uint64_t L = df;
    for (uint32_t i = 0; i < level; i++) {
        if (L <= TOPK_TILE) return 0;
        const uint64_t t1 = (L - 1) / TOPK_TILE;                  // full tiles before the last
        const uint64_t last = L - t1 * TOPK_TILE;
        L = t1 * k + (last < k ? last : k);
    }
    *len = L;
    return (uint32_t)((L + TOPK_TILE - 1) / TOPK_TILE);
}

// count[q] = min(k, df(q)) for every query of the batch
__global__ void __launch_bounds__(BLK) k_topk_count(const unsigned long long *__restrict__ off, uint32_t nq,
                                                    uint32_t k, uint32_t *count) {
    const uint64_t q = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (q >= nq) return;
    const uint64_t df = off[q + 1] - off[q];
    count[q] = df < k ? (uint32_t)df : k;
}

// The emit walk of k_dlist on the queries [q0, q0 + nqr) alone: item starts and entry offsets relative to
// the round's first item i0 and first entry e0.
__global__ void __launch_bounds__(BLK) k_topk_rebase(const unsigned long long *__restrict__ item_start,
                                                     const unsigned long long *__restrict__ item_off, uint32_t q0,
                                                     uint32_t nqr, uint64_t i0, uint64_t items, uint64_t e0,
                                                     unsigned long long *start_out, unsigned long long *off_out) {
    const uint64_t x = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (x <= nqr) start_out[x] = item_start[q0 + x] - i0;
    if (x < items) off_out[x] = item_off[i0 + x] - e0;
}

// Scan input over the round's queries: their tiles at `level`.
struct TopkTileCount {
    const unsigned long long *off;
    uint32_t q0, nqr, k, level;
    __device__ uint32_t operator()(uint64_t q) const {
        if (q >= nqr) return 0u;
        uint64_t len;
        return topk_tiles(off[q0 + q + 1] - off[q0 + q], k, level, &len);
    }
};

// One warp per query of df in [1, TOPK_WARP].
__global__ void __launch_bounds__(BLK) k_topk_warp(TopkArgs P, const uint32_t *__restrict__ x) {
    const uint32_t w = (uint32_t)(((uint64_t)blockIdx.x * BLK + threadIdx.x) >> 5);
    if (w >= P.nqr) return;                                       // whole warps
    const uint32_t l = lane_id();
    const uint32_t q = P.q0 + w;
    const uint64_t df = P.off[q + 1] - P.off[q];
    if (df == 0 || df > TOPK_WARP) return;
    const uint64_t o = P.off[q] - P.e0;
    unsigned long long key = l < df ? topk_key(P, x[o + l], x[P.R + o + l]) : 0ull;
    for (uint32_t size = 2; size <= 32; size <<= 1) {             // bitonic, descending across the lanes
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            const unsigned long long other = __shfl_xor_sync(FULL, key, stride);
            const bool keep_max = ((l & stride) == 0) == ((l & size) == 0);
            key = keep_max ? (key > other ? key : other) : (key < other ? key : other);
        }
    }
    if (l < df && l < P.k) topk_put(P, (uint64_t)q * P.k + l, key);
}

// One block per tile of `level` (grid-stride over *ntiles).  FIRST reads the listing in x, later levels
// the keys in src; a query of more than one tile writes candidates to dst, one of a single tile its answer.
template <bool FIRST>
__global__ void __launch_bounds__(BLK) k_topk_tile(TopkArgs P, uint32_t level, const uint32_t *__restrict__ tile_start,
                                                   const uint32_t *__restrict__ ntiles, const uint32_t *__restrict__ x,
                                                   const unsigned long long *__restrict__ src,
                                                   unsigned long long *dst) {
    __shared__ unsigned long long s_key[TOPK_TILE];
    __shared__ unsigned long long s_top[TOPK_KMAX];
    __shared__ uint32_t s_hist[256];
    __shared__ unsigned long long s_or, s_and;
    __shared__ uint32_t s_digit, s_need, s_n;
    const uint32_t tid = threadIdx.x, total = *ntiles;
    for (uint32_t tile = blockIdx.x; tile < total; tile += gridDim.x) {
        uint32_t a = 0, b = P.nqr;                                // the last query whose first tile <= tile
        while (b - a > 1) {
            const uint32_t m = a + (b - a) / 2;
            if (tile_start[m] <= tile) a = m; else b = m;
        }
        const uint32_t q = P.q0 + a;
        uint64_t len = 0;
        const uint32_t nt = topk_tiles(P.off[q + 1] - P.off[q], P.k, level, &len);
        const uint32_t t = tile - tile_start[a];
        const uint64_t o = P.off[q] - P.e0, base = o + (uint64_t)t * TOPK_TILE;
        const uint32_t L = (uint32_t)(len - (uint64_t)t * TOPK_TILE < TOPK_TILE ? len - (uint64_t)t * TOPK_TILE
                                                                                : TOPK_TILE);
        const uint32_t kk = L < P.k ? L : P.k;
        if (L <= P.k) {                                           // every key survives
            for (uint32_t j = tid; j < L; j += BLK)
                s_top[j] = FIRST ? topk_key(P, x[base + j], x[P.R + base + j]) : src[base + j];
        } else {
            if (tid == 0) { s_or = 0ull; s_and = ~0ull; }
            __syncthreads();
            unsigned long long vor = 0ull, vand = ~0ull;
            for (uint32_t j = tid; j < L; j += BLK) {
                const unsigned long long v = FIRST ? topk_key(P, x[base + j], x[P.R + base + j]) : src[base + j];
                s_key[j] = v;
                vor |= v;
                vand &= v;
            }
            for (int d = 16; d > 0; d >>= 1) {
                vor |= __shfl_xor_sync(FULL, vor, d);
                vand &= __shfl_xor_sync(FULL, vand, d);
            }
            if (lane_id() == 0) { atomicOr(&s_or, vor); atomicAnd(&s_and, vand); }
            __syncthreads();
            // L > k >= 1 unique keys, so some bit varies; the bits above it are common to the tile
            const int hb = 63 - __clzll((long long)(s_or ^ s_and));
            unsigned long long prefix = 0ull, mask = 0ull;
            uint32_t need = P.k;
            for (int sh = hb & ~7; sh >= 0; sh -= 8) {
                s_hist[tid] = 0;                                  // BLK == 256 bins
                __syncthreads();
                for (uint32_t j = tid; j < L; j += BLK) {
                    const unsigned long long v = s_key[j];
                    if ((v & mask) == prefix) atomicAdd(&s_hist[(uint32_t)(v >> sh) & 255u], 1u);
                }
                __syncthreads();
                if (tid < 32) {                                   // the digit of the need-th largest match
                    uint32_t h[8], cnt = 0;
#pragma unroll
                    for (int j = 0; j < 8; j++) { h[j] = s_hist[255 - 8 * tid - j]; cnt += h[j]; }
                    uint32_t inc = cnt;
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) {
                        const uint32_t v = __shfl_up_sync(FULL, inc, d);
                        if (tid >= (uint32_t)d) inc += v;
                    }
                    uint32_t acc = inc - cnt;
                    if (acc < need && need <= inc) {
#pragma unroll
                        for (int j = 0; j < 8; j++) {
                            if (acc + h[j] >= need) { s_digit = 255 - 8 * tid - j; s_need = need - acc; break; }
                            acc += h[j];
                        }
                    }
                }
                __syncthreads();
                prefix |= (unsigned long long)s_digit << sh;
                mask |= 255ull << sh;
                need = s_need;
                __syncthreads();                                  // s_digit / s_need are rewritten next digit
            }
            if (tid == 0) s_n = 0;
            __syncthreads();
            for (uint32_t j = tid; j < L; j += BLK) {             // exactly k keys: (key & mask) >= the k-th's
                const unsigned long long v = s_key[j];
                if ((v & mask) >= prefix) s_top[atomicAdd(&s_n, 1u)] = v;
            }
        }
        __syncthreads();
        if (nt == 1) {                                            // the answer, sorted
            uint32_t p2 = 1;
            while (p2 < kk) p2 <<= 1;
            for (uint32_t j = kk + tid; j < p2; j += BLK) s_top[j] = 0ull;
            __syncthreads();
            for (uint32_t size = 2; size <= p2; size <<= 1) {
                for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
                    for (uint32_t i = tid; i < p2 / 2; i += BLK) {
                        const uint32_t lo = i + (i & ~(stride - 1)), hi = lo + stride;
                        const unsigned long long u = s_top[lo], v = s_top[hi];
                        if ((u < v) == ((lo & size) == 0)) { s_top[lo] = v; s_top[hi] = u; }
                    }
                    __syncthreads();
                }
            }
            for (uint32_t j = tid; j < kk; j += BLK) topk_put(P, (uint64_t)q * P.k + j, s_top[j]);
        } else {
            for (uint32_t j = tid; j < kk; j += BLK) dst[o + (uint64_t)t * P.k + j] = s_top[j];
        }
        __syncthreads();                                          // shared memory is reused by the next tile
    }
}

}  // namespace b200sa
