// classify.cuh -- the building blocks of the S/L type classification (K1, done
// by k_classify_fused in classify2.cuh and k_classify_packed in
// classify_packed.cuh), K2: bucket tables, and the text packing and access
// helpers.  Together they replace SuffixTypes::compute (reference
// src/table.rs:592-615) and Bins::find_sizes / find_*_pointers
// (src/table.rs:686-720).
//
// Layout: position i lives in bit (i & 31) of word (i >> 5).
//   stype[w]  bit set  <=> position is S-class (Ascending or Valley)
//   lmsb[w]   bit set  <=> position is a Valley (LMS)
// Algorithm: rel(i) = cmp(T[i],T[i+1]) (rel(n-1) := L, src/table.rs:602);
// type(i) = first non-EQ rel(j), j >= i.  One block owns 256 words (8192
// bytes).  The type of a shard's first position (multi-GPU summaries) takes
// two passes: pass A reduces each block to {L,S,P(ropagate)}, pass B resolves
// the carries right-to-left across blocks.
#pragma once
#include "common.cuh"

namespace b200sa {

constexpr uint32_t ST_L = 0, ST_S = 1, ST_P = 2;
constexpr int CLS_WORDS = BLK;             // words per block
constexpr int CLS_BYTES = CLS_WORDS * 32;  // 8192 text bytes per block

// A shard of a longer text (multi-GPU row, SURVEY 8e): the chars just outside
// the shard and the resolved type of the first position after it.  For a whole
// text: next_char = prev_char = -1.
struct ShardEdge {
    int32_t next_char;    // T[hi] or -1 when the shard ends the text
    int32_t prev_char;    // T[lo-1] or -1 when the shard starts the text
    uint32_t tail_carry;  // type of position hi (ST_L / ST_S / ST_P = unknown); only read when next_char >= 0
};

// Loads the 32 bytes of word w (zero beyond n) plus the following byte.
// Returns the number of valid positions in the word.
__device__ __forceinline__ uint32_t load_word(const uint8_t *__restrict__ text, uint64_t n, uint64_t w,
                                              uint32_t (&c)[8], uint32_t &nextc, bool &has_next,
                                              const ShardEdge &edge) {
    uint64_t p0 = w * 32;
    uint32_t cnt;
    if (p0 + 32 <= n) {
        const uint4 *q = reinterpret_cast<const uint4 *>(text + p0);
        uint4 a = __ldg(q), b = __ldg(q + 1);
        c[0] = a.x; c[1] = a.y; c[2] = a.z; c[3] = a.w;
        c[4] = b.x; c[5] = b.y; c[6] = b.z; c[7] = b.w;
        cnt = 32;
    } else {
        cnt = (p0 < n) ? (uint32_t)(n - p0) : 0u;
#pragma unroll
        for (int k = 0; k < 8; k++) c[k] = 0;
#pragma unroll
        for (int j = 0; j < 32; j++)
            if ((uint32_t)j < cnt) c[j >> 2] |= (uint32_t)__ldg(text + p0 + j) << ((j & 3) * 8);
    }
    has_next = (p0 + 32 < n);
    nextc = has_next ? (uint32_t)__ldg(text + p0 + 32) : 0u;
    if (!has_next && cnt > 0 && edge.next_char >= 0) {     // the shard continues in the next shard
        has_next = true;
        if (cnt == 32) nextc = (uint32_t)edge.next_char;
        else c[cnt >> 2] |= (uint32_t)edge.next_char << ((cnt & 3) * 8);
    }
    return cnt;
}

__device__ __forceinline__ uint32_t byte_of(const uint32_t (&c)[8], int j) {
    return (c[j >> 2] >> ((j & 3) * 8)) & 0xffu;
}

// lt/gt masks of rel(i) for the word's positions; rel(n-1) forced to L.
__device__ __forceinline__ void word_rel(const uint32_t (&c)[8], uint32_t cnt, uint32_t nextc, bool has_next,
                                         uint32_t &lt, uint32_t &gt) {
    lt = 0; gt = 0;
#pragma unroll
    for (int j = 0; j < 32; j++) {
        uint32_t a = byte_of(c, j);
        uint32_t b = (j < 31) ? byte_of(c, (j + 1) & 31) : nextc;
        bool valid = (uint32_t)j < cnt;
        bool last = ((uint32_t)j + 1 == cnt) && !has_next;   // position n-1
        if (valid) {
            if (last) gt |= 1u << j;
            else if (a < b) lt |= 1u << j;
            else if (a > b) gt |= 1u << j;
        }
    }
}

// "First non-P state among threads with larger index in this block", else
// ST_P.  mine = this thread's state.  s_warp: NWARP words.
__device__ __forceinline__ uint32_t first_nonp_right(uint32_t mine, uint32_t *s_warp) {
    const uint32_t l = lane_id(), w = warp_id();
    uint32_t nonp = __ballot_sync(FULL, mine != ST_P);
    uint32_t sb = __ballot_sync(FULL, mine == ST_S);
    __syncthreads();
    if (l == 0) s_warp[w] = nonp ? ((sb >> (__ffs(nonp) - 1)) & 1u) : ST_P;   // first non-P of the warp
    __syncthreads();
    uint32_t hm = (l == 31) ? 0u : (nonp & ~((2u << l) - 1u));
    if (hm) return (sb >> (__ffs(hm) - 1)) & 1u;
    for (uint32_t ww = w + 1; ww < NWARP; ww++) {
        uint32_t s = s_warp[ww];
        if (s != ST_P) return s;
    }
    return ST_P;
}

// Pass A: block state = first non-EQ rel in the block's byte range.
__global__ void __launch_bounds__(BLK) k_cls_block_state(const uint8_t *__restrict__ text, uint64_t n,
                                                         uint8_t *blk_state, ShardEdge edge) {
    __shared__ uint32_t s_warp[NWARP];
    uint64_t w = (uint64_t)blockIdx.x * CLS_WORDS + threadIdx.x;
    uint32_t c[8], nextc, lt, gt;
    bool has_next;
    uint32_t cnt = load_word(text, n, w, c, nextc, has_next, edge);
    word_rel(c, cnt, nextc, has_next, lt, gt);
    uint32_t ne = lt | gt;
    uint32_t mine = ne ? ((lt >> (__ffs(ne) - 1)) & 1u) : ST_P;
    uint32_t right = first_nonp_right(mine, s_warp);
    if (threadIdx.x == 0) blk_state[blockIdx.x] = (uint8_t)(mine != ST_P ? mine : right);
}

// Pass B (single block): carry_in[b] = first non-P state among blocks > b.
// Walks chunks of 256 block states from the right with a running carry.
__global__ void __launch_bounds__(BLK) k_cls_carry(const uint8_t *blk_state, uint32_t nb, uint8_t *carry_in,
                                                   uint32_t tail_carry) {
    __shared__ uint32_t s_warp[NWARP];
    uint32_t carry = tail_carry;   // whole text: unused (position n-1 is never EQ); shard: type of position hi
    uint32_t nchunks = (nb + BLK - 1) / BLK;
    for (uint32_t ch = nchunks; ch-- > 0;) {
        uint32_t b = ch * BLK + threadIdx.x;
        uint32_t mine = (b < nb) ? blk_state[b] : ST_P;
        uint32_t right = first_nonp_right(mine, s_warp);
        if (b < nb) carry_in[b] = (uint8_t)(right != ST_P ? right : carry);
        // new carry = first non-P of this chunk (thread 0's view including itself)
        __syncthreads();
        if (threadIdx.x == 0) s_warp[0] = (mine != ST_P) ? mine : (right != ST_P ? right : carry);
        __syncthreads();
        carry = s_warp[0];
        __syncthreads();
    }
}

// K2: bucket tables from the histogram (single block).
//   bstart[c] = start of bucket c in SA (bstart[256] = n)
//   Lcnt/Scnt = type-split bucket sizes, lms_off = LMS group offsets,
//   code_of[c] = rank of byte c among the bytes that occur (order preserving),
//   alpha[code] = byte, *sigma = number of distinct bytes.
__global__ void __launch_bounds__(BLK) k_bucket_tables(const uint32_t *hist768, uint32_t *bstart, uint32_t *Lcnt,
                                                       uint32_t *Scnt, uint32_t *lms_off, uint32_t *code_of,
                                                       uint32_t *alpha, uint32_t *sigma) {
    __shared__ uint32_t s_w[NWARP + 1];
    uint32_t c = threadIdx.x;
    uint32_t L = hist768[c], S = hist768[256 + c] + hist768[512 + c], M = hist768[512 + c];
    Lcnt[c] = L; Scnt[c] = S;
    uint32_t total;
    uint32_t inc = block_incl_scan<OpSum>(L + S, s_w, &total);
    bstart[c] = inc - (L + S);
    if (c == 255) bstart[256] = total;
    inc = block_incl_scan<OpSum>(M, s_w, &total);
    lms_off[c] = inc - M;
    if (c == 255) lms_off[256] = total;
    uint32_t present = (L + S) > 0 ? 1u : 0u;
    inc = block_incl_scan<OpSum>(present, s_w, &total);
    uint32_t code = inc - present;
    code_of[c] = code;
    alpha[c] = 0;
    __syncthreads();
    if (present) alpha[code] = c;
    if (c == 0) *sigma = total;
}

// Which byte values occur (for b200sa_lcp_dev, which has no classification): hist256[b] = 1 for present
// bytes -- k_alpha_from_hist only asks "> 0".  16 bytes per load; every byte stores a flag to shared memory
// (one byte extract + one store: a bit set in registers costs eight selects per byte and made the kernel
// instruction-bound at a third of the HBM bandwidth; equal flags in one word are not bank conflicts).
// gate (may be null): run only when *gate != 0.
__global__ void __launch_bounds__(BLK) k_byte_hist(const uint8_t *__restrict__ text, uint64_t n, uint32_t *hist256,
                                                   const uint32_t *gate) {
    if (gate && *gate == 0u) return;
    __shared__ uint8_t s_seen[256];
    s_seen[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t nv = n / 16;
    for (uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x; i < nv; i += (uint64_t)gridDim.x * BLK) {
        uint4 v = __ldg(reinterpret_cast<const uint4 *>(text) + i);
        uint32_t wds[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int q = 0; q < 4; q++) {
            uint32_t x = wds[q];
            s_seen[x & 0xffu] = 1; s_seen[(x >> 8) & 0xffu] = 1; s_seen[(x >> 16) & 0xffu] = 1; s_seen[x >> 24] = 1;
        }
    }
    if (blockIdx.x == 0) for (uint64_t i = nv * 16 + threadIdx.x; i < n; i += BLK) s_seen[__ldg(text + i)] = 1;
    __syncthreads();
    if (s_seen[threadIdx.x]) hist256[threadIdx.x] = 1u;
}
__global__ void __launch_bounds__(BLK) k_alpha_from_hist(const uint32_t *hist256, uint32_t *code_of, uint32_t *alpha,
                                                         uint32_t *sigma, const uint32_t *gate) {
    if (gate && *gate == 0u) return;                 // gate (may be null): as in k_byte_hist
    __shared__ uint32_t s_w[NWARP + 1];
    uint32_t c = threadIdx.x, total;
    uint32_t present = hist256[c] > 0 ? 1u : 0u;
    uint32_t inc = block_incl_scan<OpSum>(present, s_w, &total);
    uint32_t code = inc - present;
    code_of[c] = code;
    alpha[c] = 0;
    __syncthreads();
    if (present) alpha[code] = c;
    if (c == 0) *sigma = total;
}

// ---- packed text: BITS in {2,4} bits per char (dense order-preserving codes),
// 32/BITS chars per u32 word, char i at bit (i % CPW) * BITS.  BITS == 8 is the
// raw byte text.  Small alphabets make the text L2-resident (100 MB DNA ->
// 25 MB), which turns the random T[s-1] gathers of the induce into L2 hits.
// Device-side conditions (each may be null), for packing before the host has read the alphabet:
//   d_sigma  pack only when *d_sigma fits BITS;
//   gate     pack only when *gate != 0;
//   present  the codes come from the bytes flagged here (k_byte_hist of a sample of the text); a byte
//            without a flag sets *d_miss, and the words that hold it are not valid.
template <int BITS>
__global__ void __launch_bounds__(BLK) k_pack(const uint8_t *__restrict__ text, uint64_t n,
                                              const uint32_t *__restrict__ code_of, uint32_t *packed,
                                              const uint32_t *d_sigma, const uint32_t *gate,
                                              const uint32_t *present, uint32_t *d_miss) {
    constexpr int CPW = 32 / BITS;
    if (gate && *gate == 0u) return;
    if (d_sigma && *d_sigma > (1u << BITS)) return;
    __shared__ uint8_t s_lut[256];
    s_lut[threadIdx.x] = (uint8_t)(code_of[threadIdx.x] | (present && present[threadIdx.x] == 0u ? 0x80u : 0u));
    __syncthreads();
    uint64_t w = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    uint64_t p0 = w * CPW;
    if (p0 >= n) return;
    uint32_t out = 0, any = 0;                       // any: OR of the table entries (bit 7: a byte without a code)
    constexpr uint32_t MASK = (1u << BITS) - 1u;
    if (p0 + CPW <= n) {
        if (CPW == 16) {
            uint4 v = __ldg(reinterpret_cast<const uint4 *>(text + p0));
            uint32_t q[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 16; j++) {
                uint32_t e = s_lut[(q[j >> 2] >> ((j & 3) * 8)) & 0xffu];
                any |= e;
                out |= (e & MASK) << (j * BITS);
            }
        } else {
            uint2 v = __ldg(reinterpret_cast<const uint2 *>(text + p0));
            uint32_t q[2] = {v.x, v.y};
#pragma unroll
            for (int j = 0; j < 8; j++) {
                uint32_t e = s_lut[(q[j >> 2] >> ((j & 3) * 8)) & 0xffu];
                any |= e;
                out |= (e & MASK) << (j * BITS);
            }
        }
    } else {
        for (int j = 0; j < CPW && p0 + j < n; j++) {
            uint32_t e = s_lut[__ldg(text + p0 + j)];
            any |= e;
            out |= (e & MASK) << (j * BITS);
        }
    }
    packed[w] = out;
    if (d_miss && (any & 0x80u)) *d_miss = 1u;
}

template <int BITS>
__device__ __forceinline__ uint32_t text_get(const void *__restrict__ base, uint32_t i) {
    if (BITS == 8) return (uint32_t)__ldg(reinterpret_cast<const uint8_t *>(base) + i);
    constexpr int CPW = 32 / (BITS == 8 ? 4 : BITS);
    return (__ldg(reinterpret_cast<const uint32_t *>(base) + i / CPW) >> ((i % CPW) * BITS)) & ((1u << BITS) - 1u);
}

// 32 bits of packed text starting at char position pos (BITS < 8): CPW chars,
// char pos in the low bits.  Reads word w and w+1 (the packed buffer carries
// one padding word).
template <int BITS>
__device__ __forceinline__ uint32_t text_bits(const void *__restrict__ base, uint32_t pos) {
    constexpr int CPW = 32 / BITS;
    const uint32_t *pk = reinterpret_cast<const uint32_t *>(base);
    uint32_t w = pos / CPW, off = (pos % CPW) * BITS;
    uint32_t lo = __ldg(pk + w), hi = __ldg(pk + w + 1);
    return __funnelshift_r(lo, hi, off);
}
// Number of equal leading chars of text[a..) and text[b..), at most `limit`.
template <int BITS>
__device__ __forceinline__ uint32_t text_match(const void *__restrict__ base, uint32_t a, uint32_t b, uint32_t limit) {
    uint32_t done = 0;
    if (BITS == 8) {
        const uint8_t *t = reinterpret_cast<const uint8_t *>(base);
        while (done < limit && __ldg(t + a + done) == __ldg(t + b + done)) done++;
        return done;
    } else {
        constexpr int PB = (BITS == 8 ? 4 : BITS);
        constexpr int CPW = 32 / PB;
        // the common case ends inside the first word
        if (limit >= (uint32_t)CPW) {
            uint32_t x = text_bits<PB>(base, a) ^ text_bits<PB>(base, b);      // (one 16-byte load per side was slower)
            if (x) return (uint32_t)(__ffs(x) - 1) / PB;
            done = CPW;
        }
        // long matches (runs, repeats): four words per side in flight per iteration,
        // so the loop is not one L2 round trip per word
        while (done + 4 * CPW <= limit) {
            uint32_t x0 = text_bits<PB>(base, a + done) ^ text_bits<PB>(base, b + done);
            uint32_t x1 = text_bits<PB>(base, a + done + CPW) ^ text_bits<PB>(base, b + done + CPW);
            uint32_t x2 = text_bits<PB>(base, a + done + 2 * CPW) ^ text_bits<PB>(base, b + done + 2 * CPW);
            uint32_t x3 = text_bits<PB>(base, a + done + 3 * CPW) ^ text_bits<PB>(base, b + done + 3 * CPW);
            if (x0) return done + (uint32_t)(__ffs(x0) - 1) / PB;
            if (x1) return done + CPW + (uint32_t)(__ffs(x1) - 1) / PB;
            if (x2) return done + 2 * CPW + (uint32_t)(__ffs(x2) - 1) / PB;
            if (x3) return done + 3 * CPW + (uint32_t)(__ffs(x3) - 1) / PB;
            done += 4 * CPW;
        }
        while (done < limit) {
            uint32_t x = text_bits<PB>(base, a + done) ^ text_bits<PB>(base, b + done);
            uint32_t take = limit - done < (uint32_t)CPW ? limit - done : (uint32_t)CPW;
            uint32_t mask = take == (uint32_t)CPW ? 0xffffffffu : ((1u << (take * PB)) - 1u);
            x &= mask;
            if (x) return done + (uint32_t)(__ffs(x) - 1) / PB;
            done += take;
        }
        return done;
    }
}
// Warp-cooperative continuation of a long match: all 32 lanes call with the SAME
// (a, b, limit); lane l compares chars [done + l*W, done + (l+1)*W) per sweep (W =
// four words), so one sweep covers 32*W chars with coalesced loads instead of one
// lane walking word by word through two private cache-line streams.
template <int BITS>
__device__ __forceinline__ uint32_t text_match_warp(const void *__restrict__ base, uint32_t a, uint32_t b,
                                                    uint32_t limit) {
    const uint32_t l = lane_id();
    if (BITS == 8) {
        const uint8_t *t = reinterpret_cast<const uint8_t *>(base);
        uint32_t done = 0;
        while (done < limit) {
            uint32_t off = done + l * 4u, first = 0xffffffffu;
#pragma unroll
            for (int q = 3; q >= 0; q--) {
                uint32_t o = off + q;
                if (o < limit && __ldg(t + a + o) != __ldg(t + b + o)) first = o;
            }
            uint32_t m = __ballot_sync(FULL, first != 0xffffffffu);
            if (m) return __shfl_sync(FULL, first, __ffs(m) - 1);
            done += 128u;
        }
        return limit;
    } else {
        constexpr int PB = (BITS == 8 ? 4 : BITS);
        constexpr uint32_t CPW = 32 / PB, W = 4 * CPW;
        uint32_t done = 0;
        while (done < limit) {
            uint32_t off = done + l * W, first = 0xffffffffu;
#pragma unroll
            for (int q = 3; q >= 0; q--) {
                uint32_t o = off + q * CPW;
                if (o < limit) {
                    uint32_t x = text_bits<PB>(base, a + o) ^ text_bits<PB>(base, b + o);
                    uint32_t take = limit - o < CPW ? limit - o : CPW;
                    if (take < CPW) x &= (1u << (take * PB)) - 1u;
                    if (x) first = o + (uint32_t)(__ffs(x) - 1) / PB;
                }
            }
            uint32_t m = __ballot_sync(FULL, first != 0xffffffffu);
            if (m) return __shfl_sync(FULL, first, __ffs(m) - 1);
            done += 32u * W;
        }
        return limit;
    }
}

// Distance from LMS position p to the next LMS position (> p), or 0 if none.
__device__ __forceinline__ uint32_t next_lms_dist(const uint32_t *__restrict__ lmsb, uint32_t n, uint32_t p) {
    uint32_t q = p + 1;
    uint32_t nw = (n + 31) >> 5;
    uint32_t w = q >> 5;
    if (w >= nw) return 0;
    uint32_t bits = __ldg(lmsb + w) >> (q & 31);
    if (bits) return 1u + (uint32_t)(__ffs(bits) - 1);
    uint32_t dist = 1u + (32u - (q & 31));
    for (w = w + 1; w < nw; w++) {
        bits = __ldg(lmsb + w);
        if (bits) return dist + (uint32_t)(__ffs(bits) - 1);
        dist += 32;
    }
    return 0;
}

// rank of an LMS position among LMS positions in text order
__device__ __forceinline__ uint32_t lms_text_rank(const uint32_t *__restrict__ lmsb,
                                                  const uint32_t *__restrict__ lmsrank, uint32_t pos) {
    uint32_t w = pos >> 5;
    return __ldg(lmsrank + w) + __popc(__ldg(lmsb + w) & ((1u << (pos & 31)) - 1u));
}
__device__ __forceinline__ uint32_t bit_at(const uint32_t *__restrict__ bm, uint32_t pos) {
    return (__ldg(bm + (pos >> 5)) >> (pos & 31)) & 1u;
}

}  // namespace b200sa
