// common.cuh -- block/warp primitives, generic scan / compaction / radix pass.
// sm_90a only.  All kernels assume blockDim.x == BLK (256).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200sa {

constexpr int BLK = 256;            // threads per block (== radix, one thread per digit)
constexpr int NWARP = BLK / 32;
constexpr int ITEMS = 8;            // items per thread in a ranking tile
constexpr int TILE = BLK * ITEMS;   // 2048 items per tile
constexpr uint32_t FULL = 0xffffffffu;

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ uint32_t warp_id() { return threadIdx.x >> 5; }
__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

// Lanes of the warp that hold the same NBITS-bit key (and are valid), built from
// NBITS+1 ballots.  MATCH.ANY iterates over the distinct values of a warp (up to
// 32 for random digits); the ballot form is a fixed, short sequence.  Ballots
// win on random bytes, lose on 4-symbol DNA and cost registers in k_induce, so
// MATCH stays the default.
#ifndef PEERS_MATCH
#define PEERS_MATCH 1
#endif
// Peers among the lanes in `peers` (all lanes valid: pass FULL and skip the validity ballot).
template <int NBITS>
__device__ __forceinline__ uint32_t peer_mask_ballot_in(uint32_t key, uint32_t peers) {
#pragma unroll
    for (int b = 0; b < NBITS; b++) {
        bool bit = (key >> b) & 1u;
        uint32_t bal = __ballot_sync(FULL, bit);
        peers &= bit ? bal : ~bal;
    }
    return peers;
}
template <int NBITS>
__device__ __forceinline__ uint32_t peer_mask_ballot(uint32_t key, bool valid) {
    return peer_mask_ballot_in<NBITS>(key, __ballot_sync(FULL, valid));
}
template <int NBITS>
__device__ __forceinline__ uint32_t peer_mask(uint32_t key, bool valid) {
#if PEERS_MATCH
    return __match_any_sync(FULL, valid ? key : 0xffffffffu) & __ballot_sync(FULL, valid);
#else
    return peer_mask_ballot<NBITS>(key, valid);
#endif
}

// ---------------------------------------------------------------- scan ops
struct OpSum {
    using T = uint32_t;
    __device__ __forceinline__ static uint32_t id() { return 0u; }
    __device__ __forceinline__ static uint32_t op(uint32_t a, uint32_t b) { return a + b; }
};
struct OpSum64 {                    // sums that may pass 2^32 (document listing totals)
    using T = unsigned long long;
    __device__ __forceinline__ static T id() { return 0ull; }
    __device__ __forceinline__ static T op(T a, T b) { return a + b; }
};
struct OpMax {
    using T = uint32_t;
    __device__ __forceinline__ static uint32_t id() { return 0u; }
    __device__ __forceinline__ static uint32_t op(uint32_t a, uint32_t b) { return a > b ? a : b; }
};

// pair scan: max over the high word, sum over the low word (group start + active count in one pass)
struct OpMaxSum {
    using T = unsigned long long;
    __device__ __forceinline__ static T id() { return 0ull; }
    __device__ __forceinline__ static T op(T a, T b) {
        uint32_t ah = (uint32_t)(a >> 32), bh = (uint32_t)(b >> 32);
        return ((T)(ah > bh ? ah : bh) << 32) | (uint32_t)((uint32_t)a + (uint32_t)b);
    }
};

template <class Op>
__device__ __forceinline__ typename Op::T warp_incl_scan(typename Op::T v) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        typename Op::T t = __shfl_up_sync(FULL, v, o);
        if ((int)lane_id() >= o) v = Op::op(v, t);
    }
    return v;
}

// Block-wide inclusive scan of one value per thread.  s_w: NWARP+1 words of
// shared memory.  Returns the inclusive result; *total gets the block total.
template <class Op>
__device__ __forceinline__ typename Op::T block_incl_scan(typename Op::T v, typename Op::T *s_w, typename Op::T *total) {
    typedef typename Op::T T;
    T inc = warp_incl_scan<Op>(v);
    __syncthreads();                       // protect s_w from a previous use
    if (lane_id() == 31) s_w[warp_id()] = inc;
    __syncthreads();
    if (threadIdx.x == 0) {
        T run = Op::id();
        for (int w = 0; w < NWARP; w++) {
            T t = s_w[w];
            s_w[w] = run;                  // exclusive prefix of warp w
            run = Op::op(run, t);
        }
        s_w[NWARP] = run;
    }
    __syncthreads();
    *total = s_w[NWARP];
    return Op::op(s_w[warp_id()], inc);
}

// ------------------------------------------------------- generic device scan
// Three-kernel reduce / scan-partials / apply over N elements given by an
// input functor In(i) -> u32.  Out(i, exclusive, value) consumes the result.
// Each block owns a contiguous chunk of SCAN_CHUNK elements.
constexpr int SCAN_IPT = 16;
constexpr int SCAN_CHUNK = BLK * SCAN_IPT;   // 4096

template <class Op, class InF>
__global__ void __launch_bounds__(BLK) k_scan_reduce(InF in, uint64_t n, typename Op::T *partial) {
    typedef typename Op::T T;
    __shared__ T s_w[NWARP + 1];
    uint64_t base = (uint64_t)blockIdx.x * SCAN_CHUNK;
    T acc = Op::id();
#pragma unroll 4
    for (int k = 0; k < SCAN_IPT; k++) {
        uint64_t i = base + (uint64_t)k * BLK + threadIdx.x;
        if (i < n) acc = Op::op(acc, in(i));
    }
    T total;
    block_incl_scan<Op>(acc, s_w, &total);
    if (threadIdx.x == 0) partial[blockIdx.x] = total;
}

// Single block: in-place exclusive scan of partial[0..nb); total -> *out_total.
template <class Op>
__global__ void __launch_bounds__(BLK) k_scan_partials(typename Op::T *partial, uint32_t nb, typename Op::T *out_total) {
    typedef typename Op::T T;
    __shared__ T s_w[NWARP + 1];
    T carry = Op::id();
    for (uint32_t b0 = 0; b0 < nb; b0 += BLK) {
        uint32_t i = b0 + threadIdx.x;
        T v = i < nb ? partial[i] : Op::id();
        T total;
        T inc = block_incl_scan<Op>(v, s_w, &total);
        T prev = __shfl_up_sync(FULL, inc, 1);
        T exc = (lane_id() == 0) ? s_w[warp_id()] : prev;       // exclusive prefix inside the chunk
        if (i < nb) partial[i] = Op::op(carry, exc);
        carry = Op::op(carry, total);
        __syncthreads();
    }
    if (threadIdx.x == 0 && out_total) *out_total = carry;
}

// Warp-blocked layout: warp w owns SCAN_IPT*32 consecutive elements of the
// chunk, read in SCAN_IPT coalesced rounds of 32; each round is one warp scan
// with a running carry, then one cross-warp fix-up.
template <class Op, class InF, class OutF>
__global__ void __launch_bounds__(BLK) k_scan_apply(InF in, OutF out, uint64_t n, const typename Op::T *partial_excl) {
    typedef typename Op::T T;
    __shared__ T s_w[NWARP + 1];
    const uint32_t w = warp_id(), l = lane_id();
    uint64_t base = (uint64_t)blockIdx.x * SCAN_CHUNK + (uint64_t)w * (SCAN_IPT * 32) + l;
    T v[SCAN_IPT], exc[SCAN_IPT];
    T carry = Op::id();
#pragma unroll
    for (int k = 0; k < SCAN_IPT; k++) {
        uint64_t i = base + (uint64_t)k * 32;
        v[k] = (i < n) ? (T)in(i) : Op::id();
        T inc = warp_incl_scan<Op>(v[k]);
        T prev = __shfl_up_sync(FULL, inc, 1);
        exc[k] = Op::op(carry, l == 0 ? Op::id() : prev);
        carry = Op::op(carry, __shfl_sync(FULL, inc, 31));
    }
    if (l == 0) s_w[w] = carry;           // warp total
    __syncthreads();
    if (threadIdx.x == 0) {
        T run = partial_excl[blockIdx.x];
        for (int ww = 0; ww < NWARP; ww++) {
            T t = s_w[ww];
            s_w[ww] = run;
            run = Op::op(run, t);
        }
    }
    __syncthreads();
    T wbase = s_w[w];
#pragma unroll
    for (int k = 0; k < SCAN_IPT; k++) {
        uint64_t i = base + (uint64_t)k * 32;
        if (i < n) out(i, Op::op(wbase, exc[k]), v[k]);
    }
}

// ---------------------------------------------------- single-pass device scan
// Decoupled look-back (one kernel, the input is read ONCE): tiles are claimed in
// order through an atomic ticket; a tile publishes its aggregate, warp 0 walks
// back over the predecessors' descriptors (32 at a time) until it meets an
// inclusive prefix, publishes its own inclusive prefix and the block applies it.
// Descriptor per tile: agg (u64), incl (u64), flag (u32).  Flags are epoch-tagged
// (epoch+1 = aggregate ready, epoch+2 = inclusive ready; the host bumps the epoch
// by 2 per scan), so the descriptor arrays never need clearing between scans; the
// ticket is reset by the block that draws the last tile.  Value before flag with a
// gpu-scope fence in between on the writer side, flag before value on the reader
// side.  All ops used here are commutative and associative.
__device__ __forceinline__ uint32_t ld_relaxed_u32(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u32(uint32_t *p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long *p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
template <class T>
__device__ __forceinline__ T shfl_t(T v, int src) { return __shfl_sync(FULL, v, src); }

struct ScanState {
    unsigned long long *agg;     // [tiles]
    unsigned long long *incl;    // [tiles]
    uint32_t *flag;              // [tiles]
    unsigned long long *pk;      // [tiles] packed descriptors of the u32-sum look-back: (epoch + state) << 32 | value
    uint32_t *ticket;            // [1], zero between kernels
    uint32_t epoch;
};

// Warp-0 part of a tile, in two halves so that a kernel can put independent work between them
// (the walk is short once the predecessors had time to publish inclusive prefixes):
//   tile_publish  -- one lane publishes the tile aggregate;
//   tile_walk     -- all 32 lanes of ONE warp walk back over the predecessors (32 at a time) until an
//                    inclusive prefix, publish this tile's inclusive prefix and return the exclusive one
//                    (in every lane).  `last` = this is the final tile (writes *d_total).
template <class Op>
__device__ __forceinline__ void tile_publish(const ScanState &S, uint32_t tile, typename Op::T block_total) {
    if (tile > 0) {
        st_relaxed_u64(S.agg + tile, (unsigned long long)block_total);
        __threadfence();
        st_relaxed_u32(S.flag + tile, S.epoch + 1u);
    }
}
template <class Op>
__device__ __forceinline__ typename Op::T tile_walk(const ScanState &S, uint32_t tile, typename Op::T block_total,
                                                    bool last, typename Op::T *d_total) {
    typedef typename Op::T T;
    const uint32_t l = lane_id();
    T prefix = Op::id();
    if (tile > 0) {
        int64_t t0 = (int64_t)tile - 1;
        while (true) {
            int64_t tt = t0 - (int64_t)l;            // lane 0: nearest predecessor
            uint32_t st = 2u;                         // before tile 0: inclusive prefix = identity
            T val = Op::id();
            if (tt >= 0) {
                uint32_t f;
                do { f = ld_relaxed_u32(S.flag + tt) - S.epoch; } while (f != 1u && f != 2u);
                __threadfence();
                st = f;
                val = (T)ld_relaxed_u64((f == 2u ? S.incl : S.agg) + tt);
            }
            uint32_t im = __ballot_sync(FULL, st == 2u);
            uint32_t first = im ? (uint32_t)(__ffs(im) - 1) : 32u;
            T contrib = (l <= first) ? val : Op::id();
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) contrib = Op::op(contrib, __shfl_xor_sync(FULL, contrib, o));
            prefix = Op::op(prefix, contrib);
            if (im) break;
            t0 -= 32;
        }
    }
    if (l == 0) {
        T total = Op::op(prefix, block_total);
        st_relaxed_u64(S.incl + tile, (unsigned long long)total);
        __threadfence();
        st_relaxed_u32(S.flag + tile, S.epoch + 2u);
        if (last && d_total) *d_total = total;
    }
    return prefix;
}
// The same two halves for u32 SUMS with the descriptor in ONE 64-bit word (state tag | value): a window of
// 32 predecessors costs one load round trip instead of flag -> fence -> value, and publishing is one
// store.  Kernels whose tiles are short (the fused classifier: 12 k tiles of 8 KB) run at the speed of
// this chain -- every wave of resident tiles waits for inclusive prefixes to travel through it.
__device__ __forceinline__ void tile_publish_u32(const ScanState &S, uint32_t tile, uint32_t block_total) {
    if (tile > 0) st_relaxed_u64(S.pk + tile, ((unsigned long long)(S.epoch + 1u) << 32) | block_total);
}
constexpr int LB_K = 1;      // descriptors per lane and round trip: the walk looks at 32 * K predecessors at once (K = LB_K
                             // unless the kernel asks for more)
template <int K = LB_K>
__device__ __forceinline__ uint32_t tile_walk_u32(const ScanState &S, uint32_t tile, uint32_t block_total, bool last,
                                                  uint32_t *d_total) {
    const uint32_t l = lane_id();
    uint32_t prefix = 0;
    if (tile > 0) {
        // A tile publishes its inclusive prefix only when its own walk ends, so a walk has to cross every
        // predecessor that is still in flight; with w predecessors per round trip the chain moves w tiles
        // per L2 latency, and kernels with short tiles run at exactly that speed: one-word descriptors
        // beat flag -> fence -> value even with w = 32 on the fused classifier.
        const unsigned long long before = ((unsigned long long)(S.epoch + 2u) << 32);   // "tile -1": inclusive 0
        int64_t t0 = (int64_t)tile - 1;
        bool done = false;
        while (!done) {
            unsigned long long v[K];
#pragma unroll
            for (int j = 0; j < K; j++) {           // nearest predecessors in v[0] (lane 0 nearest)
                int64_t tt = t0 - (int64_t)(l + 32u * j);
                v[j] = tt >= 0 ? ld_relaxed_u64(S.pk + tt) : before;
            }
#pragma unroll
            for (int j = 0; j < K; j++) {
                if (done) break;
                int64_t tt = t0 - (int64_t)(l + 32u * j);
                uint32_t st = (uint32_t)(v[j] >> 32) - S.epoch;
                while (st != 1u && st != 2u) { v[j] = ld_relaxed_u64(S.pk + tt); st = (uint32_t)(v[j] >> 32) - S.epoch; }
                uint32_t im = __ballot_sync(FULL, st == 2u);
                uint32_t first = im ? (uint32_t)(__ffs(im) - 1) : 32u;
                prefix += __reduce_add_sync(FULL, (l <= first) ? (uint32_t)v[j] : 0u);
                done = im != 0u;
            }
            t0 -= 32 * K;
        }
    }
    if (l == 0) {
        uint32_t total = prefix + block_total;
        st_relaxed_u64(S.pk + tile, ((unsigned long long)(S.epoch + 2u) << 32) | total);
        if (last && d_total) *d_total = total;
    }
    return prefix;
}
template <class Op>
__device__ __forceinline__ typename Op::T tile_lookback(const ScanState &S, uint32_t tile, typename Op::T block_total,
                                                        bool last, typename Op::T *d_total) {
    if (lane_id() == 0) tile_publish<Op>(S, tile, block_total);
    return tile_walk<Op>(S, tile, block_total, last, d_total);
}

template <class Op, class InF, class OutF>
__global__ void __launch_bounds__(BLK) k_scan_lb(InF in, OutF out, uint64_t n, uint32_t ntiles, ScanState S,
                                                 typename Op::T *d_total) {
    typedef typename Op::T T;
    __shared__ T s_w[NWARP + 1];
    __shared__ uint32_t s_tile;
    if (threadIdx.x == 0) {
        uint32_t t = atomicAdd(S.ticket, 1u);
        if (t + 1 == ntiles) *S.ticket = 0u;         // every tile has been drawn: re-arm for the next kernel
        s_tile = t;
    }
    __syncthreads();
    const uint32_t tile = s_tile, w = warp_id(), l = lane_id();
    const uint64_t base = (uint64_t)tile * SCAN_CHUNK + (uint64_t)w * (SCAN_IPT * 32) + l;
    T v[SCAN_IPT], exc[SCAN_IPT];
#pragma unroll
    for (int k = 0; k < SCAN_IPT; k++) {
        uint64_t i = base + (uint64_t)k * 32;
        v[k] = (i < n) ? (T)in(i) : Op::id();
    }
    T carry = Op::id();
#pragma unroll
    for (int k = 0; k < SCAN_IPT; k++) {
        T inc = warp_incl_scan<Op>(v[k]);
        T prev = __shfl_up_sync(FULL, inc, 1);
        exc[k] = Op::op(carry, l == 0 ? Op::id() : prev);
        carry = Op::op(carry, shfl_t(inc, 31));
    }
    if (l == 0) s_w[w] = carry;           // warp totals
    __syncthreads();
    if (w == 0) {
        T t = (l < (uint32_t)NWARP) ? s_w[l] : Op::id();
        T inc = warp_incl_scan<Op>(t);
        const T block_total = shfl_t(inc, NWARP - 1);
        T prevw = __shfl_up_sync(FULL, inc, 1);
        T wexc = (l == 0) ? Op::id() : prevw;          // exclusive prefix of warp l inside the block
        T prefix = tile_lookback<Op>(S, tile, block_total, tile + 1 == ntiles, d_total);
        if (l < (uint32_t)NWARP) s_w[l] = Op::op(prefix, wexc);
    }
    __syncthreads();
    const T wbase = s_w[w];
#pragma unroll
    for (int k = 0; k < SCAN_IPT; k++) {
        uint64_t i = base + (uint64_t)k * 32;
        if (i < n) out(i, Op::op(wbase, exc[k]), v[k]);
    }
}

// ------------------------------------------------------------- tile ranking
// Stable multi-way ranking of one tile (TILE items, warp-blocked layout:
// warp w, round r, lane l owns logical item  w*ITEMS*32 + r*32 + l).
// dig[r] in [0,256) for valid items.  Requires s_wcnt[NWARP][256] zeroed and a
// __syncthreads() before the call.  After the call (which ends with a
// __syncthreads()):  position of item = digit_base[d] + s_wcnt[w][d] + rank[r]
// and s_tcnt[d] = number of valid items with digit d in the tile.
template <int N>
__device__ __forceinline__ void tile_rank(const uint32_t (&dig)[N], uint32_t validmask,
                                          uint32_t (&rank)[N],
                                          uint32_t (*s_wcnt)[256], uint32_t *s_tcnt) {
    const uint32_t w = warp_id();
    const uint32_t lt = lanemask_lt();
#pragma unroll
    for (int r = 0; r < N; r++) {
        bool valid = (validmask >> r) & 1u;
        uint32_t peers = peer_mask<8>(dig[r], valid);
        uint32_t below = __popc(peers & lt);
        uint32_t base = valid ? s_wcnt[w][dig[r]] : 0u;
        __syncwarp();
        if (valid && below == 0) s_wcnt[w][dig[r]] = base + __popc(peers);
        __syncwarp();
        rank[r] = base + below;
    }
    __syncthreads();
    {
        uint32_t d = threadIdx.x;      // BLK == 256 digits
        uint32_t run = 0;
#pragma unroll
        for (int ww = 0; ww < NWARP; ww++) {
            uint32_t t = s_wcnt[ww][d];
            s_wcnt[ww][d] = run;
            run += t;
        }
        s_tcnt[d] = run;
    }
    __syncthreads();
}

// Warp-aggregated shared-memory histogram increment (all 32 lanes must call).
template <int NBITS = 8>
__device__ __forceinline__ void hist_add(uint32_t *s_hist, uint32_t key, bool valid) {
    uint32_t peers = peer_mask<NBITS>(key, valid);
    if (valid && (peers & lanemask_lt()) == 0) atomicAdd(&s_hist[key], (uint32_t)__popc(peers));
}

// Same aggregation into a histogram that is PRIVATE to the calling warp: the
// leader lanes hold distinct keys, so a plain read-modify-write replaces the
// shared-memory atomic (ATOMS is issued once per lane).
template <int NBITS = 8>
__device__ __forceinline__ void hist_add_private(uint32_t *s_warp_hist, uint32_t key, bool valid) {
    uint32_t peers = peer_mask<NBITS>(key, valid);
    if (valid && (peers & lanemask_lt()) == 0) s_warp_hist[key] += (uint32_t)__popc(peers);
    __syncwarp();
}

// Ballot-built peer mask variant for near-random 8-bit digits (radix-sort
// histograms): fixed 9 ballots instead of a MATCH that iterates over up to 32
// distinct values.
__device__ __forceinline__ void hist_add_private_ballot(uint32_t *s_warp_hist, uint32_t key, bool valid) {
    uint32_t peers = peer_mask_ballot<8>(key, valid);
    if (valid && (peers & lanemask_lt()) == 0) s_warp_hist[key] += (uint32_t)__popc(peers);
    __syncwarp();
}

// ------------------------------------------------------------ radix passes
// One stable LSD pass over N items whose 8-bit digit is DigF(i); MoveF(i,dst)
// moves item i to output slot dst.  Block b owns tiles [b*tpb, (b+1)*tpb).
// cnt layout: cnt[d*nb + b] (digit-major) so that one exclusive scan over the
// whole array yields global bases.
template <class DigF>
__global__ void __launch_bounds__(BLK) k_radix_hist(DigF dig, uint64_t n, uint32_t tpb, uint32_t *cnt) {
    __shared__ uint32_t s_hist[256];
    s_hist[threadIdx.x] = 0;
    __syncthreads();
    uint64_t t0 = (uint64_t)blockIdx.x * tpb * TILE;
    uint64_t t1 = t0 + (uint64_t)tpb * TILE;
    if (t1 > n) t1 = n;
    // round up so that every lane of every warp executes hist_add together
    for (uint64_t i0 = t0; i0 < t1; i0 += BLK) {
        uint64_t i = i0 + threadIdx.x;
        bool valid = i < t1;
        uint32_t d = valid ? dig(i) : 0u;
        hist_add(s_hist, d, valid);
    }
    __syncthreads();
    cnt[(uint64_t)threadIdx.x * gridDim.x + blockIdx.x] = s_hist[threadIdx.x];
}

template <class DigF, class MoveF>
__global__ void __launch_bounds__(BLK) k_radix_scatter(DigF dig, MoveF mv, uint64_t n, uint32_t tpb,
                                                       const uint32_t *cnt_excl) {
    __shared__ uint32_t s_wcnt[NWARP][256];
    __shared__ uint32_t s_tcnt[256];
    __shared__ uint32_t s_base[256];
    s_base[threadIdx.x] = cnt_excl[(uint64_t)threadIdx.x * gridDim.x + blockIdx.x];
    uint64_t t0 = (uint64_t)blockIdx.x * tpb * TILE;
    uint64_t t1 = t0 + (uint64_t)tpb * TILE;
    if (t1 > n) t1 = n;
    const uint32_t w = warp_id(), l = lane_id();
    for (uint64_t tb = t0; tb < t1; tb += TILE) {
#pragma unroll
        for (int ww = 0; ww < NWARP; ww++) s_wcnt[ww][threadIdx.x] = 0;
        __syncthreads();
        uint32_t d[ITEMS], rank[ITEMS], vm = 0;
#pragma unroll
        for (int r = 0; r < ITEMS; r++) {
            uint64_t i = tb + (uint64_t)w * (ITEMS * 32) + r * 32 + l;
            bool valid = i < t1;
            d[r] = valid ? dig(i) : 0u;
            vm |= (valid ? 1u : 0u) << r;
        }
        tile_rank(d, vm, rank, s_wcnt, s_tcnt);
#pragma unroll
        for (int r = 0; r < ITEMS; r++) {
            if ((vm >> r) & 1u) {
                uint64_t i = tb + (uint64_t)w * (ITEMS * 32) + r * 32 + l;
                uint32_t dst = s_base[d[r]] + s_wcnt[w][d[r]] + rank[r];
                mv(i, dst);
            }
        }
        __syncthreads();
        s_base[threadIdx.x] += s_tcnt[threadIdx.x];
        __syncthreads();
    }
}

}  // namespace b200sa

// ---------------------------------------------------------------- one-sweep LSD radix sort
// (key,u32 value) pairs, 8-bit digits.  One upfront kernel builds the digit
// histograms of ALL passes; each pass then reads the data once: tiles are
// claimed in order through an atomic ticket, per-tile digit counts are chained
// with decoupled look-back (64-bit status words: flag in bits 62-63, count in
// the low 32), and the tile is staged through shared memory in digit order so
// that the global writes are contiguous runs.
namespace b200sa {

constexpr unsigned long long OS_AGG = 1ull << 62, OS_INCL = 2ull << 62, OS_VAL = 0xffffffffull;
// status words are self-contained (flag + count in one 64-bit word), so relaxed
// gpu-scope accesses suffice; they avoid the system-scope LDG of `volatile`.
__device__ __forceinline__ unsigned long long os_load(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void os_store(unsigned long long *p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
constexpr int OS_MAX_PASSES = 8;

// dynamic shared memory: [NWARP][npass][256] u32 (64 KB for 8 passes)
template <class K, class KeyF>
__global__ void __launch_bounds__(BLK) k_os_hist(KeyF keyf, uint64_t n, int npass, uint32_t shift0, uint32_t *ghist,
                                                 K *keys_out = nullptr) {
    extern __shared__ uint32_t s_dyn[];
    const uint32_t w = warp_id();
    for (int i = threadIdx.x; i < NWARP * npass * 256; i += BLK) s_dyn[i] = 0;
    __syncthreads();
    uint32_t *mine = s_dyn + (size_t)w * npass * 256;
    // four keys per thread in flight (the key functor may gather: position -> text window); digit
    // counts go to the warp's private histograms with shared-memory atomics (cheaper than 9
    // ballots per digit)
    for (uint64_t i0 = (uint64_t)blockIdx.x * (BLK * 4); i0 < n; i0 += (uint64_t)gridDim.x * (BLK * 4)) {
        K key[4];
        bool valid[4];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            uint64_t i = i0 + (uint64_t)q * BLK + threadIdx.x;
            valid[q] = i < n;
            key[q] = valid[q] ? keyf(i) : (K)0;
            if (keys_out && valid[q]) keys_out[i] = key[q];       // gathered keys: the first pass reads them back in order
        }
#pragma unroll
        for (int q = 0; q < 4; q++)
            if (valid[q])
                for (int p = 0; p < npass; p++) atomicAdd(&mine[p * 256 + ((uint32_t)(key[q] >> (shift0 + 8 * p)) & 0xffu)], 1u);
    }
    __syncthreads();
    for (int p = 0; p < npass; p++) {
        uint32_t v = 0;
#pragma unroll
        for (int ww = 0; ww < NWARP; ww++) v += s_dyn[((size_t)ww * npass + p) * 256 + threadIdx.x];
        if (v) atomicAdd(&ghist[p * 256 + threadIdx.x], v);
    }
}

// digit bases when the keys are a permutation of 0..n-1 and the digit is their
// top byte: bin d holds exactly the keys [d << shift, (d+1) << shift)
__global__ void __launch_bounds__(BLK) k_os_perm_base(uint32_t *gbase, uint32_t shift, uint32_t n) {
    uint64_t b = (uint64_t)threadIdx.x << shift;
    gbase[threadIdx.x] = b < n ? (uint32_t)b : n;
}
// one block per pass: exclusive scan of its 256 digit totals, in place
__global__ void __launch_bounds__(BLK) k_os_scan(uint32_t *ghist) {
    __shared__ uint32_t s_w[NWARP + 1];
    uint32_t v = ghist[blockIdx.x * 256 + threadIdx.x], total;
    uint32_t inc = block_incl_scan<OpSum>(v, s_w, &total);
    ghist[blockIdx.x * 256 + threadIdx.x] = inc - v;
}

#ifndef OS_MINB
#define OS_MINB 4
#endif
template <class K>
struct LoadArr {
    const K *a;
    __device__ __forceinline__ K operator()(uint64_t i) const { return a[i]; }
    __device__ __forceinline__ K at(uint64_t i, uint32_t) const { return a[i]; }     // key of item i given its value
};
// OSI items per thread: 8 (tile of 2048) for small sorts; the wide tiles (32 keys per thread for 32-bit keys, 16 for
// 64-bit keys) take two CTAs per SM and keep every key, value and the look-back word in registers without spills.
#ifndef OS_MINB_WIDE
#define OS_MINB_WIDE 2
#endif
// dynamic shared memory of k_os_pass: the tile's keys and values in digit order
template <class K, int OSI>
constexpr size_t os_stage_bytes() { return (size_t)OSI * BLK * (sizeof(K) + sizeof(uint32_t)); }
// One stable pass.  The tile's digit counts are known before any item is ranked: each warp counts its digits
// with shared-memory atomics, the counts are published at once (tile 0 publishes them as inclusive), and the
// load of the nearest predecessor's status word is in flight while the warps rank their items.  Ranking
// builds each item's peers from 9 ballots (MATCH.ANY iterates over the ~30 distinct digits a warp holds on
// random keys) and seeds a running (warp, digit) counter with the warp's offset inside the tile; the leader
// of each peer group advances it with one atomic and hands the old value to its peers by shuffle.  Items go
// straight to their slot in the staging arrays; the look-back then ends on the first inclusive prefix.
template <class K, class KeyF, class ValF, int OSI = ITEMS>
__global__ void __launch_bounds__(BLK, (OSI > 8 ? OS_MINB_WIDE : OS_MINB)) k_os_pass(KeyF keyf, ValF valf, K *kout,
                                                 uint32_t *vout, uint64_t n, uint32_t shift,
                                                 const uint32_t *__restrict__ gbase, volatile unsigned long long *status,
                                                 uint32_t *ticket) {
    __shared__ uint32_t s_wcnt[NWARP][256];
    __shared__ uint32_t s_gb[256];
    __shared__ uint32_t s_w[NWARP + 1];
    __shared__ uint32_t s_tile;
    extern __shared__ __align__(16) unsigned char s_os_stage[];
    K *s_k = reinterpret_cast<K *>(s_os_stage);
    uint32_t *s_v = reinterpret_cast<uint32_t *>(s_k + OSI * BLK);
    if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
#pragma unroll
    for (int ww = 0; ww < NWARP; ww++) s_wcnt[ww][threadIdx.x] = 0;
    __syncthreads();
    const uint32_t tile = s_tile, w = warp_id(), l = lane_id();
    const uint64_t tb = (uint64_t)tile * (OSI * BLK);
    const bool full = tb + OSI * BLK <= n;      // every tile but the last: no bounds, no validity ballot
    K key[OSI];
    uint32_t val[OSI], vm = 0;
#pragma unroll
    for (int r = 0; r < OSI; r++) {             // all values first: a key functor that gathers through the value
        uint64_t i = tb + (uint64_t)w * (OSI * 32) + r * 32 + l;   // (position -> text window) then has its eight
        bool valid = full || i < n;                                   // dependent loads in flight together
        val[r] = valid ? valf(i) : 0u;
        vm |= (valid ? 1u : 0u) << r;
    }
#pragma unroll
    for (int r = 0; r < OSI; r++) {
        uint64_t i = tb + (uint64_t)w * (OSI * 32) + r * 32 + l;
        key[r] = ((vm >> r) & 1u) ? keyf.at(i, val[r]) : (K)0;
    }
    auto digit = [&](int r) { return (uint32_t)(key[r] >> shift) & 0xffu; };
#pragma unroll
    for (int r = 0; r < OSI; r++)
        if ((vm >> r) & 1u) atomicAdd(&s_wcnt[w][digit(r)], 1u);
    __syncthreads();
    const uint32_t dg = threadIdx.x;
    const uint32_t gb = gbase[dg];
    uint32_t c[NWARP], cnt = 0;
#pragma unroll
    for (int ww = 0; ww < NWARP; ww++) {
        c[ww] = s_wcnt[ww][dg];
        cnt += c[ww];
    }
    unsigned long long *st = const_cast<unsigned long long *>(status);
    os_store(st + (uint64_t)tile * 256 + dg, (tile == 0 ? OS_INCL : OS_AGG) | cnt);
    int64_t t = (int64_t)tile - 1;
    unsigned long long x = t >= 0 ? os_load(st + (uint64_t)t * 256 + dg) : OS_INCL;
    uint32_t total;
    const uint32_t texcl = block_incl_scan<OpSum>(cnt, s_w, &total) - cnt;
    {
        uint32_t run = texcl;             // column dg is read and written by thread dg only
#pragma unroll
        for (int ww = 0; ww < NWARP; ww++) {
            s_wcnt[ww][dg] = run;
            run += c[ww];
        }
    }
    __syncthreads();
    const uint32_t lt = lanemask_lt();
#pragma unroll
    for (int r = 0; r < OSI; r++) {
        bool valid = (vm >> r) & 1u;
        uint32_t peers = peer_mask_ballot_in<8>(digit(r), full ? FULL : __ballot_sync(FULL, valid));
        uint32_t below = __popc(peers & lt), old = 0;
        if (valid && below == 0) old = atomicAdd(&s_wcnt[w][digit(r)], (uint32_t)__popc(peers));
        uint32_t p = __shfl_sync(FULL, old, __ffs(peers) - 1) + below;
        if (valid) {
            s_k[p] = key[r];
            s_v[p] = val[r];
        }
    }
    // tile 0 is inclusive from the start, so the walk never passes it
    uint32_t excl = 0;
    while (true) {
        while ((x >> 62) == 0) x = os_load(st + (uint64_t)t * 256 + dg);
        excl += (uint32_t)(x & OS_VAL);
        if ((x >> 62) == 2) break;
        t--;
        x = os_load(st + (uint64_t)t * 256 + dg);
    }
    if (tile > 0) os_store(st + (uint64_t)tile * 256 + dg, OS_INCL | (unsigned long long)(excl + cnt));
    s_gb[dg] = gb + excl - texcl;
    __syncthreads();
    uint64_t left = n - tb;
    uint32_t cnt_tile = left < (uint64_t)(OSI * BLK) ? (uint32_t)left : (uint32_t)(OSI * BLK);
    auto put = [&](uint32_t j) {
        K k = s_k[j];
        uint32_t dst = s_gb[(uint32_t)(k >> shift) & 0xffu] + j;
        kout[dst] = k;
        vout[dst] = s_v[j];
    };
    if (full) {
#pragma unroll
        for (int r = 0; r < OSI; r++) put(r * BLK + threadIdx.x);
    } else {
        for (uint32_t j = threadIdx.x; j < cnt_tile; j += BLK) put(j);
    }
}

}  // namespace b200sa
