// classify2.cuh -- K1 fused: ONE pass over the text produces the S/L type bitmap, the LMS
// bitmap, the (byte, L / S / LMS) histogram and the LMS positions (in DESCENDING text order,
// the order the LMS sort is fed in).  Replaces SuffixTypes::compute (reference
// src/table.rs:592-615), Bins::find_sizes (:686-704) and the LMS position fill (P15,
// :512-520).  It classifies every text whose bytes are not classified from 2-bit packed
// words (classify_packed.cuh), and every shard of a multi-GPU build.
//
// type(i) = first non-equal cmp(T[j], T[j+1]), j >= i, so information flows right to left:
// tiles (8192 bytes) are claimed from the END of the text through an atomic ticket.  A tile
// publishes its own state {L, S, P(ropagate)} at once; only a tile that consists of one
// repeated byte up to its end has to wait for a state further right (decoupled look-back
// over epoch-tagged status words).  The LMS positions of a tile go to
// lmspos_desc[#LMS to the right of the tile ...], a sum look-back in the same direction, so
// the whole classification is a single kernel that reads the text once.
// Per-word work is SWAR: byte compares four at a time, type bits by a 5-step segmented
// fill, histogram by warp-uniform candidate bytes (popcounts of SWAR equality masks) with a
// shared-memory atomic tail for large alphabets.
#pragma once
#include "classify.cuh"

namespace b200sa {

// bit k of the result = most significant bit of byte k of x
__device__ __forceinline__ uint32_t msb4(uint32_t x) {
    return (((x & 0x80808080u) >> 7) * 0x01020408u) >> 24;        // low 4 bits
}
// 0x80 in every byte of x that is zero (exact, no borrow artefacts)
__device__ __forceinline__ uint32_t zero_bytes(uint32_t x) {
    uint32_t t = (x & 0x7f7f7f7fu) + 0x7f7f7f7fu;
    return ~(t | x | 0x7f7f7f7fu);
}
// mask of the positions of the 32-byte word c whose byte equals v
__device__ __forceinline__ uint32_t eq_mask32(const uint32_t (&c)[8], uint32_t v) {
    const uint32_t rep = v * 0x01010101u;
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) m |= (msb4(zero_bytes(c[k] ^ rep)) & 0xfu) << (4 * k);
    return m;
}
// lt / gt masks of cmp(T[j], T[j+1]) for the 32 positions of a word (SWAR form of word_rel)
__device__ __forceinline__ void word_rel_swar(const uint32_t (&c)[8], uint32_t cnt, uint32_t nextc, bool has_next,
                                              uint32_t &lt, uint32_t &gt) {
    lt = 0; gt = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        uint32_t a = c[k];
        uint32_t b = (c[k] >> 8) | ((k < 7 ? c[k + 1] : nextc) << 24);
        lt |= (msb4(__vcmpltu4(a, b)) & 0xfu) << (4 * k);
        gt |= (msb4(__vcmpgtu4(a, b)) & 0xfu) << (4 * k);
    }
    uint32_t vmask = (cnt >= 32) ? 0xffffffffu : ((1u << cnt) - 1u);
    lt &= vmask; gt &= vmask;
    if (!has_next && cnt > 0) {               // position n-1 is L by definition (src/table.rs:602)
        uint32_t bit = 1u << (cnt - 1);
        lt &= ~bit; gt |= bit;
    }
}
// S-type bits of a word: bit j = lt at the first position k >= j with lt|gt set, else cin
__device__ __forceinline__ uint32_t resolve_types(uint32_t lt, uint32_t gt, uint32_t cin) {
    uint32_t m = __brev(lt | gt), v = __brev(lt);
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
        v |= (v << s) & ~m;
        m |= m << s;
    }
    if (cin) v |= ~m;
    return __brev(v);
}

constexpr uint32_t HIST_COPIES = 64;
// hist[k] = sum of the interleaved copies
__global__ void __launch_bounds__(BLK) k_hist_fold(const uint32_t *__restrict__ copies, uint32_t *hist) {
    for (uint32_t k = threadIdx.x; k < 768; k += BLK) {
        uint32_t v = 0;
        for (uint32_t q = 0; q < HIST_COPIES; q++) v += copies[(size_t)q * 768u + k];
        hist[k] = v;
    }
}

struct Cls2State {
    uint32_t *state;     // [tiles] epoch-tagged: tag + 1 + {ST_L, ST_S, ST_P}
    uint32_t tag;        // distinct per call
};

__global__ void __launch_bounds__(BLK) k_classify_fused(const uint8_t *__restrict__ text, uint64_t n, uint32_t ntiles,
                                                        ScanState S, Cls2State CS, uint32_t *stype, uint32_t *lmsb,
                                                        uint32_t *hist768, uint32_t *lmspos_desc, uint32_t *d_m,
                                                        ShardEdge edge, const uint32_t *d_sigma_packed) {
    // d_sigma_packed (may be null): the device-side alphabet size when k_classify_packed was launched too;
    // 2-bit text is its job, so every block returns before it takes a ticket
    if (d_sigma_packed && *d_sigma_packed <= 4u) return;
    __shared__ uint32_t s_warp[NWARP];
    __shared__ uint32_t s_sw[BLK];
    __shared__ uint32_t s_hist[NWARP][768];
    __shared__ __align__(128) uint32_t s_lms[CLS_BYTES / 2];      // the tile's LMS positions, descending
    __shared__ uint32_t s_w[NWARP + 1];
    __shared__ uint32_t s_tile, s_carry, s_prefix;
    const uint32_t tid = threadIdx.x, wp = warp_id(), l = lane_id();
    if (tid == 0) {
        uint32_t t = atomicAdd(S.ticket, 1u);
        if (t + 1 == ntiles) *S.ticket = 0u;
        s_tile = t;
    }
    for (int k = tid; k < NWARP * 768; k += BLK) (&s_hist[0][0])[k] = 0;
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint64_t cb = (uint64_t)(ntiles - 1u - tile);            // tiles are claimed from the end of the text
    const uint64_t w = cb * CLS_WORDS + tid;
    const uint64_t nw = (n + 31) / 32;
    uint32_t c[8], nextc, lt, gt;
    bool has_next;
    uint32_t cnt = load_word(text, n, w, c, nextc, has_next, edge);
    word_rel_swar(c, cnt, nextc, has_next, lt, gt);
    uint32_t ne = lt | gt;
    uint32_t mine = ne ? ((lt >> (__ffs(ne) - 1)) & 1u) : ST_P;
    uint32_t right = first_nonp_right(mine, s_warp);
    // ---- publish the tile's own state; fetch the carry from the right if any word needs it
    if (tid == 0) {
        uint32_t st = (mine != ST_P) ? mine : right;
        st_relaxed_u32(CS.state + tile, CS.tag + 1u + st);
        uint32_t carry = (edge.next_char >= 0) ? edge.tail_carry : ST_L;     // beyond the text / shard
        for (int64_t tt = (int64_t)tile - 1; tt >= 0; tt--) {
            uint32_t v;
            do { v = ld_relaxed_u32(CS.state + tt) - CS.tag - 1u; } while (v > 2u);
            if (v != ST_P) { carry = v; break; }
        }
        s_carry = carry;
        // a tile of one repeated byte republishes the RESOLVED state, so that tiles further
        // left stop here instead of walking over every such tile again (runs of equal bytes)
        if (st == ST_P) st_relaxed_u32(CS.state + tile, CS.tag + 1u + carry);
    }
    __syncthreads();
    uint32_t cin = (right != ST_P) ? right : s_carry;
    uint32_t vmask = (cnt >= 32) ? 0xffffffffu : ((1u << cnt) - 1u);
    uint32_t sw = resolve_types(lt, gt, cin == ST_S ? 1u : 0u) & vmask;
    s_sw[tid] = sw;
    __syncthreads();
    uint32_t pb;                                      // type bit of the position just before this word
    if (tid > 0) pb = s_sw[tid - 1] >> 31;
    else if (w == 0 && edge.prev_char < 0) pb = 1u;   // position 0 is never a Valley (src/table.rs:465)
    else if (w == 0) {
        uint32_t c1 = (uint32_t)edge.prev_char, c2 = c[0] & 0xffu;
        pb = (c1 < c2) ? 1u : (c1 > c2) ? 0u : (sw & 1u);
    } else if (cnt == 0) pb = 0u;
    else {
        uint32_t c1 = __ldg(text + w * 32 - 1), c2 = c[0] & 0xffu;
        pb = (c1 < c2) ? 1u : (c1 > c2) ? 0u : (sw & 1u);
    }
    uint32_t lw = sw & ~((sw << 1) | pb);
    if (w < nw) { stype[w] = sw; lmsb[w] = lw; }
    // ---- LMS positions: rank from the right
    uint32_t nl = __popc(lw), btot;
    uint32_t inc = block_incl_scan<OpSum>(nl, s_w, &btot);
    uint32_t suf = btot - inc;                        // LMS positions in the words to the right inside the tile
    {
        uint32_t bits = lw, k = suf;
        while (bits) {
            uint32_t j = 31u - (uint32_t)__clz(bits);
            bits &= ~(1u << j);
            s_lms[k++] = (uint32_t)(w * 32 + j);
        }
    }
    if (tid == 0) tile_publish_u32(S, tile, btot);       // the walk follows the histogram: by then the
                                                            // predecessors have published inclusive prefixes
    // ---- histogram: warp-uniform candidate bytes first (small alphabets finish here)
    {
        uint32_t mM = lw, mS = sw & ~lw, mL = ~sw & vmask, todo = vmask;
        uint32_t *h = s_hist[wp];
        for (int it = 0; it < 6; it++) {
            uint32_t prop = todo ? ((c[(__ffs(todo) - 1) >> 2] >> (((__ffs(todo) - 1) & 3) * 8)) & 0xffu) : 0xffffffffu;
            uint32_t cand = __reduce_min_sync(FULL, prop);
            if (cand == 0xffffffffu) break;
            uint32_t eq = eq_mask32(c, cand) & todo;
            todo &= ~eq;
            uint32_t tL = __reduce_add_sync(FULL, (uint32_t)__popc(eq & mL));
            uint32_t tS = __reduce_add_sync(FULL, (uint32_t)__popc(eq & mS));
            uint32_t tM = __reduce_add_sync(FULL, (uint32_t)__popc(eq & mM));
            if (l == 0) { h[cand] += tL; h[256 + cand] += tS; h[512 + cand] += tM; }
            __syncwarp();
        }
        while (todo) {                                 // large alphabets: the rest one by one
            uint32_t j = __ffs(todo) - 1;
            todo &= todo - 1;
            uint32_t cls = ((sw >> j) & 1u) + ((lw >> j) & 1u);
            atomicAdd(&h[((c[j >> 2] >> ((j & 3) * 8)) & 0xffu) + 256u * cls], 1u);
        }
    }
    __syncthreads();
    // warp 0 walks the look-back chain; meanwhile the other warps flush the tile's histogram.  12 k tiles
    // adding to the same few global words serialise in L2 (measured), so HIST_COPIES interleaved copies
    // are summed by k_hist_fold
    if (wp == 0) {
        uint32_t prefix = tile_walk_u32(S, tile, btot, tile + 1 == ntiles, d_m);
        if (l == 0) s_prefix = prefix;
    } else {
        uint32_t *hcopy = hist768 + (size_t)(tile % HIST_COPIES) * 768u;
        for (int k = tid - 32; k < 768; k += BLK - 32) {
            uint32_t v = 0;
#pragma unroll
            for (int ww = 0; ww < NWARP; ww++) v += s_hist[ww][k];
            if (v) atomicAdd(&hcopy[k], v);
        }
    }
    __syncthreads();
    if (lmspos_desc) {
        const uint32_t base = s_prefix;
        for (uint32_t k = tid; k < btot; k += BLK) lmspos_desc[base + k] = s_lms[k];
    }
}

// ascending copy for the consumers that want text order (robust path, shard API)
__global__ void __launch_bounds__(BLK) k_reverse_u32(const uint32_t *__restrict__ in, uint32_t m, uint32_t *out) {
    uint32_t i = blockIdx.x * BLK + threadIdx.x;
    if (i < m) out[i] = in[m - 1u - i];
}

}  // namespace b200sa
