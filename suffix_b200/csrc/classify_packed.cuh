// classify_packed.cuh -- the fused classification (classify2.cuh) of 2-bit packed text, plus the first
// window key of every LMS suffix.  One pass over the packed words produces the S/L type bitmap, the LMS
// bitmap, the (byte, L / S / LMS) histogram, the LMS positions in DESCENDING text order and, next to each,
// its 16-character window key as lms_window<2> computes it, together with the digit histograms of key bits
// 16-31 -- so the LMS sort starts at its first one-sweep pass instead of gathering the windows again
// (k_os_hist).  A packed word holds 16 characters, so a thread classifies 128 characters from 32 bytes and
// a tile covers 32768 characters: a quarter of the byte classifier's look-back chain.
#pragma once
#include "classify2.cuh"
#include "lms_sort.cuh"

namespace b200sa {

constexpr int CP_WORDS = 8;                                    // packed words per thread
constexpr int CP_TILE_WORDS = BLK * CP_WORDS;                  // 2048 packed words per tile
constexpr uint32_t CP_TILE_CHARS = (uint32_t)CP_TILE_WORDS * 16u;   // 32768 characters per tile
constexpr int CP_LB = 4;                                       // look-back descriptors per lane and round trip

// even bits of x to the low half, odd bits to the high half (inverse perfect shuffle): of a packed word,
// the low code bits of its 16 characters and their high code bits
__device__ __forceinline__ uint32_t unzip_bits(uint32_t x) {
    uint32_t t;
    t = (x ^ (x >> 1)) & 0x22222222u; x ^= t ^ (t << 1);
    t = (x ^ (x >> 2)) & 0x0c0c0c0cu; x ^= t ^ (t << 2);
    t = (x ^ (x >> 4)) & 0x00f000f0u; x ^= t ^ (t << 4);
    t = (x ^ (x >> 8)) & 0x0000ff00u; x ^= t ^ (t << 8);
    return x;
}

// Tiles are claimed from the end of the text with the ticket, chained by the epoch-tagged Cls2State carry
// and ranked by the one-word look-back, exactly as in k_classify_fused.  Runs only when *d_sigma <= 4 (the
// text was packed at 2 bits by k_pack<2> from the same device-side sigma); otherwise every block returns
// before it takes a ticket and k_classify_fused classifies the bytes.
//   alpha:   dense code -> byte (T_ALPHA), to fold the code histogram into the byte histogram
//   keys:    keys[i] = window key of lmsdesc[i]
//   ghist:   digit counts of key bits 16-23 in [0, 256) and of bits 24-31 in [256, 512), zeroed before
__global__ void __launch_bounds__(BLK) k_classify_packed(const uint32_t *__restrict__ packed, uint64_t n, uint32_t ntiles,
                                                         const uint32_t *d_sigma, const uint32_t *__restrict__ alpha,
                                                         ScanState S, Cls2State CS, uint32_t *stype, uint32_t *lmsb,
                                                         uint32_t *hist768, uint32_t *lmsdesc, uint32_t *keys,
                                                         uint32_t *ghist, uint32_t *d_m) {
    __shared__ uint32_t s_warp[NWARP];
    __shared__ uint32_t s_sw[BLK];
    __shared__ uint32_t s_wd[CP_TILE_WORDS + 1];                // the tile's packed words + the first one to its right
    __shared__ uint16_t s_off[CP_TILE_CHARS / 2];               // LMS offsets inside the tile, descending
    __shared__ uint32_t s_dig[2][256];
    __shared__ uint32_t s_cnt[12];                              // [class * 4 + code]
    __shared__ uint32_t s_w[NWARP + 1];
    __shared__ uint32_t s_tile, s_carry, s_prefix;
    if (*d_sigma > 4u) return;
    const uint32_t tid = threadIdx.x, l = lane_id();
    if (tid == 0) {
        uint32_t t = atomicAdd(S.ticket, 1u);
        if (t + 1 == ntiles) *S.ticket = 0u;
        s_tile = t;
    }
    for (uint32_t k = tid; k < 512; k += BLK) (&s_dig[0][0])[k] = 0;
    if (tid < 12) s_cnt[tid] = 0;
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint64_t cb = (uint64_t)(ntiles - 1u - tile);            // tiles are claimed from the end of the text
    const uint64_t nwp = (n + 15) / 16, nw = (n + 31) / 32;
    const uint64_t w0 = cb * CP_TILE_WORDS + (uint64_t)tid * CP_WORDS;      // first packed word of the thread
    uint32_t x[CP_WORDS + 1];                                       // x[8]: the next thread's first word
    if (w0 + CP_WORDS <= nwp) {
        const uint4 *q = reinterpret_cast<const uint4 *>(packed + w0);
#pragma unroll
        for (int v = 0; v < CP_WORDS / 4; v++) {
            uint4 a = __ldg(q + v);
            x[4 * v] = a.x; x[4 * v + 1] = a.y; x[4 * v + 2] = a.z; x[4 * v + 3] = a.w;
        }
    } else {
#pragma unroll
        for (int k = 0; k < CP_WORDS; k++) x[k] = w0 + k < nwp ? __ldg(packed + w0 + k) : 0u;
    }
    x[CP_WORDS] = w0 + CP_WORDS < nwp ? __ldg(packed + w0 + CP_WORDS) : 0u;
#pragma unroll
    for (int k = 0; k < CP_WORDS; k++) s_wd[tid * CP_WORDS + k] = x[k];
    if (tid == BLK - 1) s_wd[CP_TILE_WORDS] = x[CP_WORDS];
    // ---- per 32-character output word: low / high code bits, lt and non-equal masks of cmp(T[j], T[j+1])
    constexpr int OW = CP_WORDS / 2;
    const uint64_t p0 = w0 * 16;
    uint32_t lo[OW], hi[OW], lt[OW], ne[OW], vm[OW];
#pragma unroll
    for (int k = 0; k < OW; k++) {
        uint32_t u0 = unzip_bits(x[2 * k]), u1 = unzip_bits(x[2 * k + 1]), nx = x[2 * k + 2];
        lo[k] = (u0 & 0xffffu) | (u1 << 16);
        hi[k] = (u0 >> 16) | (u1 & 0xffff0000u);
        uint32_t lon = (lo[k] >> 1) | (nx << 31), hin = (hi[k] >> 1) | ((nx >> 1) << 31);
        lt[k] = (~hi[k] & hin) | (~(hi[k] ^ hin) & ~lo[k] & lon);
        ne[k] = (hi[k] ^ hin) | (lo[k] ^ lon);
        const uint64_t pw = p0 + 32u * k;
        const uint32_t cnt = pw >= n ? 0u : (n - pw >= 32 ? 32u : (uint32_t)(n - pw));
        vm[k] = cnt >= 32 ? 0xffffffffu : ((1u << cnt) - 1u);
        lt[k] &= vm[k]; ne[k] &= vm[k];
        if (cnt > 0 && pw + 32 >= n) {                      // position n-1 is L by definition (src/table.rs:602)
            uint32_t bit = 1u << (cnt - 1);
            lt[k] &= ~bit; ne[k] |= bit;
        }
    }
    uint32_t mine = ST_P;
#pragma unroll
    for (int k = OW - 1; k >= 0; k--)
        if (ne[k]) mine = (lt[k] >> (__ffs(ne[k]) - 1)) & 1u;
    uint32_t right = first_nonp_right(mine, s_warp);
    // ---- publish the tile's own state; fetch the carry from the right if any word needs it
    if (tid == 0) {
        uint32_t st = (mine != ST_P) ? mine : right;
        st_relaxed_u32(CS.state + tile, CS.tag + 1u + st);
        uint32_t carry = ST_L;                                       // beyond the text
        for (int64_t tt = (int64_t)tile - 1; tt >= 0; tt--) {
            uint32_t v;
            do { v = ld_relaxed_u32(CS.state + tt) - CS.tag - 1u; } while (v > 2u);
            if (v != ST_P) { carry = v; break; }
        }
        s_carry = carry;
        if (st == ST_P) st_relaxed_u32(CS.state + tile, CS.tag + 1u + carry);
    }
    __syncthreads();
    uint32_t cin = (right != ST_P) ? right : s_carry;
    uint32_t sw[OW];
#pragma unroll
    for (int k = OW - 1; k >= 0; k--) {
        sw[k] = resolve_types(lt[k], ne[k], cin == ST_S ? 1u : 0u) & vm[k];
        cin = sw[k] & 1u;
    }
    s_sw[tid] = sw[OW - 1];
    __syncthreads();
    uint32_t pb;                                      // type bit of the position just before the thread's characters
    if (tid > 0) pb = s_sw[tid - 1] >> 31;
    else if (w0 == 0) pb = 1u;                        // position 0 is never a Valley (src/table.rs:465)
    else {
        uint32_t c1 = __ldg(packed + w0 - 1) >> 30, c2 = x[0] & 3u;
        pb = (c1 < c2) ? 1u : (c1 > c2) ? 0u : (sw[0] & 1u);
    }
    uint32_t lw[OW], nl = 0;
#pragma unroll
    for (int k = 0; k < OW; k++) {
        lw[k] = sw[k] & ~((sw[k] << 1) | pb);
        pb = sw[k] >> 31;
        nl += __popc(lw[k]);
        const uint64_t ow = w0 / 2 + k;
        if (ow < nw) { stype[ow] = sw[k]; lmsb[ow] = lw[k]; }
    }
    // ---- LMS offsets: rank from the right.  The tile's aggregate is published at once; warp 0 walks the
    // look-back chain as soon as its own offsets and counts are done, with no block barrier before.
    uint32_t btot;
    uint32_t inc = block_incl_scan<OpSum>(nl, s_w, &btot);
    if (tid == 0) tile_publish_u32(S, tile, btot);
    {
        uint32_t at = btot - inc;                     // LMS positions in the threads to the right inside the tile
#pragma unroll
        for (int k = OW - 1; k >= 0; k--) {
            uint32_t bits = lw[k];
            while (bits) {
                uint32_t j = 31u - (uint32_t)__clz(bits);
                bits &= ~(1u << j);
                s_off[at++] = (uint16_t)(tid * (CP_WORDS * 16) + 32u * k + j);
            }
        }
    }
    // ---- (code, class) counts from popcounts of the code-bit masks: of the positions in class mask M, code 3
    // has both bits, code 2 the high bit only, code 1 the low bit only
    {
        uint32_t h[12];
#pragma unroll
        for (int i = 0; i < 12; i++) h[i] = 0;
#pragma unroll
        for (int k = 0; k < OW; k++) {
            const uint32_t cls[3] = {~sw[k] & vm[k], sw[k] & ~lw[k], lw[k]};     // L, S non-LMS, LMS
#pragma unroll
            for (int q = 0; q < 3; q++) {
                uint32_t a = __popc(cls[q]), b = __popc(cls[q] & hi[k] & lo[k]);
                uint32_t hh = __popc(cls[q] & hi[k]), oo = __popc(cls[q] & lo[k]);
                h[4 * q + 3] += b; h[4 * q + 2] += hh - b; h[4 * q + 1] += oo - b; h[4 * q] += a - hh - oo + b;
            }
        }
#pragma unroll
        for (int i = 0; i < 12; i++) {
            uint32_t v = __reduce_add_sync(FULL, h[i]);
            if (l == 0 && v) atomicAdd(&s_cnt[i], v);
        }
    }
    if (warp_id() == 0) {
        uint32_t prefix = tile_walk_u32<CP_LB>(S, tile, btot, tile + 1 == ntiles, d_m);
        if (l == 0) s_prefix = prefix;
    }
    __syncthreads();
    if (warp_id() == 1 && l < 12) {                  // the counts into a histogram copy
        uint32_t v = s_cnt[l];
        if (v) atomicAdd(&hist768[(size_t)(tile % HIST_COPIES) * 768u + 256u * (l >> 2) + __ldg(alpha + (l & 3u))], v);
    }
    // ---- positions and window keys in descending order, coalesced; digit counts of key bits 16-31
    const uint32_t base = s_prefix;
    const uint64_t tbase = cb * CP_TILE_CHARS;
    for (uint32_t k = tid; k < btot; k += BLK) {
        const uint32_t off = s_off[k], wi = off >> 4;
        const uint32_t p = (uint32_t)(tbase + off);
        uint32_t xw = __funnelshift_r(s_wd[wi], s_wd[wi + 1], 2u * (off & 15u));
        const uint64_t left = n - p;
        if (left < 16) xw &= (1u << (2u * (uint32_t)left)) - 1u;
        const uint32_t key = rev_pairs(xw);
        lmsdesc[base + k] = p;
        keys[base + k] = key;
        atomicAdd(&s_dig[0][(key >> 16) & 0xffu], 1u);
        atomicAdd(&s_dig[1][key >> 24], 1u);
    }
    __syncthreads();
    {
        uint32_t v0 = s_dig[0][tid], v1 = s_dig[1][tid];
        if (v0) atomicAdd(&ghist[tid], v0);
        if (v1) atomicAdd(&ghist[256 + tid], v1);
    }
}

}  // namespace b200sa
