// lms_sort.cuh -- direct sort of the LMS suffixes ("LMS substring bucket sort" +
// "rank/rename" of the north-star pipeline, fused into one radix sort with
// refinement): replaces, for texts whose LMS suffixes are told apart by a few
// windows of characters, the reference's stage-1 machinery
//   P5  LMS into bucket tails            src/table.rs:411-416
//   P7/P9 first L/S induce               src/table.rs:421-448
//   P10 compaction, P11 naming, P12      src/table.rs:450-492 (wstring_equal :802-820)
//   P13 recursion on the reduced string  src/table.rs:494-506
//   P15/P16 un-rename                    src/table.rs:512-530
// whose only product is "the LMS suffixes in suffix order" (the seed of the final
// induce, P18, src/table.rs:536-541).
//
// Formulation.  A window key packs the next KC characters of a suffix, first
// character most significant, as a base-sigma number of dense order-preserving
// codes (sigma^KC <= 2^32; for 2-bit packed text simply the 16 two-bit codes), with
// zeros past the end of the text.
//   round 1: one-sweep LSD radix sort of (window(p), p) over all LMS positions;
//   round r: the members of groups that are still tied after (r-1)*KC characters are
//            ordered inside their group by the next window (MSD refinement; tiny
//            groups by counting, otherwise radix on (group, window)).
// End of text (src/table.rs:374: a proper prefix sorts first, there is no sentinel):
// the first sort is fed in DESCENDING text position and every later sort is stable,
// so inside a group of equal padded keys the order is always descending position.
// A member whose window runs past n ("truncated", p + h + KC > n) is a proper prefix
// of every non-truncated member with the same padded key and of every truncated
// member before which it stands, so truncated members are final exactly where the
// stable sort leaves them and each forms a group of its own.
// Texts that stay tied (long repeats: LCP >> KC * rounds) are handed to the robust
// path (stage-1 induce + naming + rank doubling); see lms_direct_sort() in b200sa.cu.
#pragma once
#include "classify.cuh"

namespace b200sa {

struct LmsWin {
    const void *ptext;            // packed words (BITS 2/4) or the byte text (BITS 8)
    const uint32_t *code_of;      // [256] dense codes (BITS 8, sigma < 256)
    uint32_t n, sigma, kc;        // kc = characters per window
};

// pair-reversal of 16 two-bit groups: char 0 (low bits) becomes the most significant
__device__ __forceinline__ uint32_t rev_pairs(uint32_t x) {
    uint32_t y = __brev(x);
    return ((y & 0x55555555u) << 1) | ((y >> 1) & 0x55555555u);
}

// window key of text[p .. p+kc), zero-padded past n;  p <= n
template <int BITS>
__device__ __forceinline__ uint32_t lms_window(const LmsWin &W, uint32_t p) {
    const uint32_t left = W.n - p;                 // valid characters from p on
    if (BITS == 2) {
        if (left == 0) return 0u;
        uint32_t x = text_bits<2>(W.ptext, p);
        if (left < 16u) x &= (1u << (2u * left)) - 1u;
        return rev_pairs(x);
    } else if (BITS == 4) {
        if (left == 0) return 0u;
        uint32_t lo = text_bits<4>(W.ptext, p);
        uint32_t hi = (W.kc > 8u && left > 8u) ? text_bits<4>(W.ptext, p + 8u) : 0u;
        uint32_t key = 0;
        for (uint32_t i = 0; i < W.kc; i++) {
            uint32_t c = (i < 8u ? (lo >> (4u * i)) : (hi >> (4u * (i - 8u)))) & 15u;
            key = key * W.sigma + (i < left ? c : 0u);
        }
        return key;
    } else {
        const uint8_t *t = reinterpret_cast<const uint8_t *>(W.ptext);
        uint32_t key = 0;
        if (W.sigma == 256u) {
#pragma unroll
            for (uint32_t i = 0; i < 4u; i++) key = (key << 8) | (i < left ? (uint32_t)__ldg(t + p + i) : 0u);
            return key;
        }
        for (uint32_t i = 0; i < W.kc; i++) {
            uint32_t c = i < left ? __ldg(W.code_of + __ldg(t + p + i)) : 0u;
            key = key * W.sigma + c;
        }
        return key;
    }
}

// first-pass functors of the one-sweep sort: item i = i-th LMS position from the END of the
// text (the fused classifier emits them in that order)
template <int BITS>
struct LmsKeyDesc {
    LmsWin W; const uint32_t *lmsdesc;
    __device__ __forceinline__ uint32_t operator()(uint64_t i) const { return lms_window<BITS>(W, __ldg(lmsdesc + i)); }
    __device__ __forceinline__ uint32_t at(uint64_t, uint32_t pos) const { return lms_window<BITS>(W, pos); }   // value = position
};
struct LmsValDesc {
    const uint32_t *lmsdesc;
    __device__ __forceinline__ uint32_t operator()(uint64_t i) const { return __ldg(lmsdesc + i); }
};

// ---- round 1: groups of equal window keys in the sorted list (slot = index).
// Only LMS positions inside the last `span` characters can be truncated (at most span/2
// of them, the first entries of the descending list).  One small kernel finds their slots -- they
// stand at the very start of their run of equal keys, in descending position -- and
// sets "forced head" bits for the slot and its successor, so that the scan over all m
// elements reads the keys only.
template <int BITS>
__global__ void __launch_bounds__(BLK) k_lms_mark_trunc(LmsWin W, const uint32_t *__restrict__ lmsdesc, uint32_t m,
                                                        const uint32_t *__restrict__ K, const uint32_t *__restrict__ P,
                                                        uint32_t span, uint32_t *forced) {
    uint32_t t = threadIdx.x;
    if (t >= m || t >= span) return;
    uint32_t p = lmsdesc[t];
    if ((uint64_t)p + span <= W.n) return;                // not truncated
    uint32_t key = lms_window<BITS>(W, p);
    uint32_t lo = 0, hi = m;
    while (lo < hi) {                                     // first slot with K >= key
        uint32_t mid = lo + (hi - lo) / 2;
        if (K[mid] < key) lo = mid + 1; else hi = mid;
    }
    for (uint32_t j = lo; j < m && K[j] == key; j++) {
        if (P[j] == p) {
            atomicOr(&forced[j >> 5], 1u << (j & 31));
            if (j + 1 < m) atomicOr(&forced[(j + 1) >> 5], 1u << ((j + 1) & 31));
            break;
        }
    }
}
// Compaction of the elements tied with a neighbour (round-1 groups): aslot / apos get the slot and the
// position, ahead[k] = slot if the element starts its group, else 0 (a max-scan over the compacted list
// turns it into the group id).  ONE specialised single-pass kernel (the generic scan with functors spent
// ~90 instructions per element on functor calls and 16 warp scans per thread): a thread owns 16
// consecutive slots, reads its 18 keys with four 16-byte loads + 2, derives heads / tied flags in
// registers and takes part in one block scan; tile offsets by the same look-back as k_scan_lb.
constexpr int LG_IPT = 16;
constexpr int LG_TILE = BLK * LG_IPT;       // 4096 slots per tile
__global__ void __launch_bounds__(BLK) k_lms_groups1(const uint32_t *__restrict__ K, const uint32_t *__restrict__ P,
                                                     const uint32_t *__restrict__ forced, uint32_t m, uint32_t ntiles,
                                                     ScanState S, uint32_t *aslot, uint32_t *apos, uint32_t *ahead,
                                                     uint32_t *d_total) {
    __shared__ uint32_t s_w[NWARP + 1];
    __shared__ uint32_t s_tile, s_prefix;
    if (threadIdx.x == 0) {
        uint32_t t = atomicAdd(S.ticket, 1u);
        if (t + 1 == ntiles) *S.ticket = 0u;
        s_tile = t;
    }
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint32_t i0 = tile * LG_TILE + threadIdx.x * LG_IPT;
    uint32_t k[LG_IPT + 2];                      // k[j+1] = K[i0 + j]; k[0] = K[i0-1]; k[17] = K[i0+16]
    if (i0 + LG_IPT <= m) {
        const uint4 *q = reinterpret_cast<const uint4 *>(K + i0);
#pragma unroll
        for (int v = 0; v < 4; v++) {
            uint4 a = __ldg(q + v);
            k[1 + 4 * v] = a.x; k[2 + 4 * v] = a.y; k[3 + 4 * v] = a.z; k[4 + 4 * v] = a.w;
        }
    } else {
#pragma unroll
        for (int j = 0; j < LG_IPT; j++) k[1 + j] = (i0 + j < m) ? __ldg(K + i0 + j) : 0u;
    }
    k[0] = (i0 > 0 && i0 <= m) ? __ldg(K + i0 - 1) : 0u;
    k[LG_IPT + 1] = (i0 + LG_IPT < m) ? __ldg(K + i0 + LG_IPT) : 0u;
    // forced-head bits of slots i0 .. i0+16 (i0 is a multiple of 16)
    uint32_t fw = (i0 < m) ? __ldg(forced + (i0 >> 5)) : 0u;
    uint32_t fbits = (fw >> (i0 & 31)) & 0xffffu;
    if (i0 + LG_IPT < m) {
        uint32_t nxt = ((i0 & 31) == 16) ? __ldg(forced + (i0 >> 5) + 1) : (fw >> 16);
        fbits |= (nxt & 1u) << 16;
    }
    uint32_t head = 0;                           // bit j: slot i0+j starts a group (bit 16: the slot after the chunk)
#pragma unroll
    for (int j = 0; j <= LG_IPT; j++) {
        uint32_t i = i0 + j;
        bool h = (i == 0) | (i >= m) | (k[j + 1] != k[j]) | ((fbits >> j) & 1u);
        head |= (h ? 1u : 0u) << j;
    }
    uint32_t act = 0;                            // bit j: slot i0+j is tied with a neighbour
#pragma unroll
    for (int j = 0; j < LG_IPT; j++) {
        bool a = (i0 + j < m) && !(((head >> j) & 1u) && ((head >> (j + 1)) & 1u));
        act |= (a ? 1u : 0u) << j;
    }
    uint32_t cnt = __popc(act), btot;
    uint32_t inc = block_incl_scan<OpSum>(cnt, s_w, &btot);
    if (warp_id() == 0) {
        if (lane_id() == 0) tile_publish_u32(S, tile, btot);
        uint32_t prefix = tile_walk_u32(S, tile, btot, tile + 1 == ntiles, d_total);
        if (lane_id() == 0) s_prefix = prefix;
    }
    __syncthreads();
    uint32_t at = s_prefix + inc - cnt;
    while (act) {
        uint32_t j = __ffs(act) - 1;
        act &= act - 1;
        uint32_t i = i0 + j;
        aslot[at] = i; apos[at] = __ldg(P + i); ahead[at] = ((head >> j) & 1u) ? i : 0u;
        at++;
    }
}

// ---- round 1 on 2-bit text: the two low key bytes and the ties in one kernel.
// On entry (K, P) are ordered by the top 16 key bits (the first 8 characters) by two one-sweep passes;
// inside such a "bucket" the pairs keep the input order (descending position).  CTA t (ticket order) owns
// the buckets whose first slot lies in [t*BS_T, (t+1)*BS_T) -- a span of at most BS_T - 1 + BS_CAP pairs
// when no bucket is longer than BS_CAP -- and sorts it stably in shared memory by (ord << 16 | low 16
// bits), ord = the bucket's index inside the span: the (K, P) order of four full passes.  Then it finds
// the tied slots (same key as a neighbour, neither of the two truncated) and compacts them in slot order
// with the one-word look-back, group id = slot of the group's head, as k_lms_groups1 + the max-scan would.
// P leaves in slot order through Pout; the sorted keys are not stored.
// A bucket longer than BS_CAP sets *d_over and its owner writes nothing: the caller reruns the four-pass sort.
// Dynamic shared memory: BS_SMEM bytes (keys u32 + two u16 index lists of BS_SPAN_MAX entries).
constexpr uint32_t BS_T = 4096;
constexpr uint32_t BS_CAP = 4096;
constexpr uint32_t BS_SPAN_MAX = BS_T + BS_CAP;              // >= BS_T - 1 + BS_CAP; index lists fit u16
constexpr uint32_t BS_ROUNDS = BS_SPAN_MAX / BLK;            // 32 rounds of BLK slots (one bit each in a u32)
constexpr size_t BS_SMEM = (size_t)BS_SPAN_MAX * (4 + 2 + 2);
constexpr uint32_t BS_BIN_MAX = 64;                          // largest bin ranked by counting (cost ~ bin size per item)
__global__ void __launch_bounds__(BLK, 3) k_lms_bucket_sort(const uint32_t *__restrict__ K, const uint32_t *__restrict__ P,
                                                            uint32_t m, uint32_t n, uint32_t kc, uint32_t ntiles,
                                                            ScanState S, uint32_t *Pout, uint32_t *aslot,
                                                            uint32_t *apos, uint32_t *ahead, uint32_t *d_total,
                                                            uint32_t *d_over) {
    extern __shared__ uint32_t s_dyn[];
    uint32_t *s_key = s_dyn;                                                   // (ord << 16) | low 16 bits
    uint16_t *s_ia = reinterpret_cast<uint16_t *>(s_dyn + BS_SPAN_MAX);       // index lists (ping-pong)
    uint16_t *s_ib = s_ia + BS_SPAN_MAX;
    __shared__ __align__(16) uint32_t s_wcnt[NWARP][256];
    __shared__ uint32_t s_base[256], s_hist[256];
    // per (round, warp) segment of the tie sweep: (max head index << 32) | count; the passes are done by then
    unsigned long long *s_seg = reinterpret_cast<unsigned long long *>(&s_wcnt[0][0]);
    __shared__ unsigned long long s_w64[NWARP + 1];
    __shared__ uint32_t s_w[NWARP + 1];
    __shared__ uint32_t s_tile, s_lo, s_hi, s_over, s_prefix;
    const uint32_t tid = threadIdx.x, w = warp_id(), l = lane_id();
    if (tid == 0) {
        uint32_t t = atomicAdd(S.ticket, 1u);
        if (t + 1 == ntiles) *S.ticket = 0u;
        s_tile = t; s_lo = m; s_hi = m; s_over = 0u;
    }
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint32_t w0 = tile * BS_T, w1 = min(w0 + BS_T, m);
    // ---- keys [w0, w0 + BS_SPAN_MAX) into shared memory in one sweep, all loads in flight: the window, the
    // end of its last bucket and every bucket-length check lie inside
    const uint32_t e = min(m, w0 + BS_SPAN_MAX);
    const uint32_t kprev = w0 > 0 ? __ldg(K + w0 - 1) >> 16 : 0xffffffffu;      // slot 0 heads its bucket
    if (e - w0 == BS_SPAN_MAX) {
        const uint4 *q = reinterpret_cast<const uint4 *>(K + w0);
        uint4 v[BS_SPAN_MAX / 4 / BLK];
#pragma unroll
        for (int k = 0; k < (int)(BS_SPAN_MAX / 4 / BLK); k++) v[k] = __ldg(q + k * BLK + tid);
#pragma unroll
        for (int k = 0; k < (int)(BS_SPAN_MAX / 4 / BLK); k++) reinterpret_cast<uint4 *>(s_key)[k * BLK + tid] = v[k];
    } else {
        for (uint32_t i = tid; i < e - w0; i += BLK) s_key[i] = __ldg(K + w0 + i);
    }
    __syncthreads();
    // ---- bucket heads of the window: the first one starts the span; each one checks its bucket's length
    for (uint32_t i = tid; i < w1 - w0; i += BLK) {
        uint32_t hi16 = s_key[i] >> 16, pr = i > 0 ? s_key[i - 1] >> 16 : kprev;
        if (pr != hi16) {
            atomicMin(&s_lo, w0 + i);
            if (w0 + i + BS_CAP < m && (s_key[i + BS_CAP] >> 16) == hi16) atomicOr(&s_over, 1u);
        }
    }
    __syncthreads();
    const bool work = s_lo < w1 && s_over == 0u;                 // block-uniform
    if (s_over && tid == 0) *d_over = 1u;
    // ---- end of the span: the first bucket head at or after w1 (at most BS_CAP - 1 slots on when no bucket
    // overflows, so inside the keys read), else m
    if (work) {
        for (uint32_t i = w1 - w0 + tid; i < e - w0; i += BLK)
            if ((s_key[i] >> 16) != (s_key[i - 1] >> 16)) atomicMin(&s_hi, w0 + i);
        __syncthreads();
    }
    const uint32_t lo = s_lo, len = work ? s_hi - lo : 0u;
    const uint32_t R = (len + BLK - 1) / BLK;                    // rounds of BLK slots, <= BS_ROUNDS
    uint32_t *sk = s_key + (lo - w0);                            // keys of the span
    uint32_t hb = 0;                                             // bit r: slot r*BLK + tid heads (bucket, then group)
    uint32_t tb = 0;                                             // bit r: slot r*BLK + tid is tied
    unsigned long long seg_total = 0;
    uint16_t *src = s_ia;
    if (work) {
        uint32_t pv[BS_ROUNDS];                      // P of the span, all loads in flight: truncated slots
#pragma unroll
        for (uint32_t r = 0; r < BS_ROUNDS; r++) {
            if (r >= R) break;                       // block-uniform
            uint32_t j = r * BLK + tid;
            pv[r] = j < len ? __ldg(P + lo + j) : 0u;
        }
        // ord = number of bucket heads at or before the slot - 1: one ballot per (round, warp) segment + one block scan
        for (uint32_t r = 0; r < R; r++) {
            uint32_t j = r * BLK + tid;
            bool h = j < len && (j == 0 || (sk[j] >> 16) != (sk[j - 1] >> 16));
            hb |= (h ? 1u : 0u) << r;
            uint32_t bal = __ballot_sync(FULL, h);
            if (l == 0) s_hist[r * NWARP + w] = __popc(bal);
        }
        __syncthreads();
        uint32_t nb;
        {
            uint32_t v = tid < R * NWARP ? s_hist[tid] : 0u;
            uint32_t inc = block_incl_scan<OpSum>(v, s_w, &nb);
            s_hist[tid] = inc - v;
        }
        __syncthreads();
        // sort key (ord << 16) | low 16 bits (< 2^29); bit 31 = truncated (p + kc > n), left out of the digits
#pragma unroll
        for (uint32_t r = 0; r < BS_ROUNDS; r++) {
            if (r >= R) break;
            uint32_t j = r * BLK + tid;
            uint32_t bal = __ballot_sync(FULL, (hb >> r) & 1u);
            uint32_t ord = s_hist[r * NWARP + w] + __popc(bal & (lanemask_lt() | (1u << l))) - 1u;
            if (j < len) sk[j] = (ord << 16) | (sk[j] & 0xffffu) | (((uint64_t)pv[r] + kc > n) ? 0x80000000u : 0u);
        }
        __syncthreads();
        // ---- the sort.  Usually one counting scatter: bin = (ord, top lb bits of the low 16), lb = 11 - bits(ord),
        // at most 2048 bins (in s_wcnt), a few slots each on random text.  The scatter (shared atomics) leaves a
        // bin in any order; every item then takes its rank inside its bin by (key, index in the span) -- the
        // order a stable sort gives.  A span with more than 1024 buckets or a bin of more than BS_BIN_MAX items
        // (repeats) takes the LSD passes below instead.
        const int ob = nb > 1 ? 32 - __clz(nb - 1) : 0;
        bool sorted = false;
        if (ob <= 10) {
            uint32_t *s_bin = &s_wcnt[0][0];
            const int lb = 11 - ob;
            for (uint32_t i = tid; i < 2048u; i += BLK) s_bin[i] = 0;
            __syncthreads();
#pragma unroll 4
            for (uint32_t j = tid; j < len; j += BLK) {
                uint32_t k = sk[j] & 0x7fffffffu;
                atomicAdd(&s_bin[((k >> 16) << lb) | ((k & 0xffffu) >> (16 - lb))], 1u);
            }
            __syncthreads();
            uint32_t c[8], sum = 0, mx = 0;
#pragma unroll
            for (int q = 0; q < 8; q++) { c[q] = s_bin[tid * 8 + q]; sum += c[q]; mx = max(mx, c[q]); }
            uint32_t tot;
            uint32_t run = block_incl_scan<OpSum>(sum, s_w, &tot) - sum;
#pragma unroll
            for (int q = 0; q < 8; q++) { s_bin[tid * 8 + q] = run; run += c[q]; }
            if (!__syncthreads_or(mx > BS_BIN_MAX)) {
                // scatter (key bits below the bin's << 13 | index in the span): unique words, so the rank inside
                // the bin is one compare per member; the two index lists hold them as u32
                uint32_t *s_pk = reinterpret_cast<uint32_t *>(s_ia);
                const uint32_t lmask = (1u << (16 - lb)) - 1u;
#pragma unroll 4
                for (uint32_t j = tid; j < len; j += BLK) {
                    uint32_t k = sk[j] & 0x7fffffffu;
                    s_pk[atomicAdd(&s_bin[((k >> 16) << lb) | ((k & 0xffffu) >> (16 - lb))], 1u)] = ((k & lmask) << 13) | j;
                }
                __syncthreads();                     // s_bin[b] = end of bin b = start of bin b + 1
                uint32_t fin[BS_ROUNDS];             // final slot << 16 | index
#pragma unroll
                for (uint32_t r = 0; r < BS_ROUNDS; r++) {
                    if (r >= R) break;
                    uint32_t j = r * BLK + tid;
                    fin[r] = 0xffffffffu;
                    if (j < len) {
                        uint32_t x = s_pk[j], k = sk[x & 0x1fffu] & 0x7fffffffu;
                        uint32_t b = ((k >> 16) << lb) | ((k & 0xffffu) >> (16 - lb));
                        uint32_t bs = b ? s_bin[b - 1] : 0u, be = s_bin[b], rank = 0;
                        for (uint32_t q = bs; q < be; q++) rank += s_pk[q] < x ? 1u : 0u;
                        fin[r] = ((bs + rank) << 16) | (x & 0x1fffu);
                    }
                }
                __syncthreads();
#pragma unroll
                for (uint32_t r = 0; r < BS_ROUNDS; r++) {
                    if (r >= R) break;
                    if (fin[r] != 0xffffffffu) s_ia[fin[r] >> 16] = (uint16_t)(fin[r] & 0xffffu);
                }
                __syncthreads();
                sorted = true;
            }
        }
        // ---- otherwise stable LSD passes over the u16 index list, 8 bits each.  The whole span is ranked at once: warp w
        // owns the C consecutive slots [w*C, (w+1)*C), one item per lane and round, and keeps (item, digit, rank
        // among the warp's items of that digit) packed in one register per round; the per-warp digit counts then
        // give the digit histogram too, so a pass reads the list once.  Peers by one ballot per digit bit that the
        // key can have (8 for the random low bytes, about 3 for the ord byte); MATCH.ANY is no faster here.
        const int kbits = 16 + (nb > 1 ? 32 - __clz(nb - 1) : 0);
        const int npass = sorted ? 0 : (kbits + 7) / 8;
        const uint32_t C = (len + NWARP * 32 - 1) / (NWARP * 32) * 32, RW = C / 32;   // RW <= BS_ROUNDS
        const uint32_t lt = lanemask_lt();
        uint16_t *dst = s_ib;
        for (int p = 0; p < npass; p++) {
            const uint32_t sh = 8u * p;
            const int dbits = min(8, kbits - 8 * p);
#pragma unroll
            for (int ww = 0; ww < NWARP; ww++) s_wcnt[ww][tid] = 0;
            __syncthreads();
            uint32_t pk[BS_ROUNDS];                  // item | digit << 13 | rank << 21  (item < 8192, rank < 1024)
#pragma unroll
            for (uint32_t r = 0; r < BS_ROUNDS; r++) {
                if (r >= RW) break;                  // warp-uniform
                uint32_t j = w * C + r * 32 + l;
                bool v = j < len;
                uint32_t it = v ? (p == 0 ? j : src[j]) : 0u;
                uint32_t d = v ? ((sk[it] & 0x7fffffffu) >> sh) & 0xffu : 0u;
                uint32_t peers = __ballot_sync(FULL, v);
#pragma unroll
                for (int b = 0; b < 8; b++) {
                    if (b >= dbits) break;           // block-uniform
                    uint32_t bal = __ballot_sync(FULL, (d >> b) & 1u);
                    peers &= ((d >> b) & 1u) ? bal : ~bal;
                }
                uint32_t below = __popc(peers & lt);
                uint32_t base = v ? s_wcnt[w][d] : 0u;
                __syncwarp();
                if (v && below == 0) s_wcnt[w][d] = base + __popc(peers);
                __syncwarp();
                pk[r] = it | (d << 13) | ((base + below) << 21);
            }
            __syncthreads();
            {                                        // digit tid: warps' exclusive counts, then the digit bases
                uint32_t run = 0;
#pragma unroll
                for (int ww = 0; ww < NWARP; ww++) {
                    uint32_t t = s_wcnt[ww][tid];
                    s_wcnt[ww][tid] = run;
                    run += t;
                }
                uint32_t tot;
                uint32_t inc = block_incl_scan<OpSum>(run, s_w, &tot);
                s_base[tid] = inc - run;
            }
            __syncthreads();
#pragma unroll
            for (uint32_t r = 0; r < BS_ROUNDS; r++) {
                if (r >= RW) break;
                if (w * C + r * 32 + l < len) {
                    uint32_t d = (pk[r] >> 13) & 0xffu;
                    dst[s_base[d] + s_wcnt[w][d] + (pk[r] >> 21)] = (uint16_t)(pk[r] & 0x1fffu);
                }
            }
            __syncthreads();
            uint16_t *t = src; src = dst; dst = t;
        }
        // ---- group heads / tied slots; per segment: tied count and the last head
        for (uint32_t r = 0; r < R; r++) {
            uint32_t j = r * BLK + tid;
            bool h = false, tl = true;
            // neighbours' keys from the lanes beside (slots j -+ 1), the warp's ends from shared memory
            uint32_t kj = j < len ? sk[src[j]] : 0u;
            uint32_t kp = __shfl_up_sync(FULL, kj, 1), kn = __shfl_down_sync(FULL, kj, 1);
            if (j < len) {                           // a truncated slot (bit 31) is a group of its own
                if (l == 0 && j > 0) kp = sk[src[j - 1]];
                if (l == 31 && j + 1 < len) kn = sk[src[j + 1]];
                h = j == 0 || kj != kp || ((kj | kp) >> 31);
                tl = j + 1 == len || kj != kn || ((kj | kn) >> 31);
            }
            bool tied = j < len && !(h && tl);
            uint32_t balh = __ballot_sync(FULL, h), balt = __ballot_sync(FULL, tied);
            hb = (hb & ~(1u << r)) | ((h ? 1u : 0u) << r);
            tb |= (tied ? 1u : 0u) << r;
            if (l == 0) {
                uint32_t last = balh ? r * BLK + w * 32 + 31 - __clz(balh) : 0u;
                s_seg[r * NWARP + w] = ((unsigned long long)last << 32) | __popc(balt);
            }
        }
        __syncthreads();
        {
            unsigned long long v = tid < R * NWARP ? s_seg[tid] : 0ull;
            unsigned long long inc = block_incl_scan<OpMaxSum>(v, s_w64, &seg_total);
            // exclusive: the max part of the inclusive value covers this segment too -- use the previous one
            unsigned long long prev = __shfl_up_sync(FULL, inc, 1);
            unsigned long long exc = l == 0 ? s_w64[w] : prev;
            __syncthreads();
            s_seg[tid] = exc;
        }
    }
    // ---- slot-order offset of the tied slots (every CTA publishes, also an empty or overflowing one): the
    // aggregate now, the walk after the P stores, so that the predecessors have time to publish theirs
    if (tid == 0) tile_publish_u32(S, tile, (uint32_t)seg_total);
    if (work) {                                      // P in slot order: the span's P (read before, in L2) through the
        uint32_t pv[BS_ROUNDS];                      // keys' shared memory, which the ties no longer need
#pragma unroll
        for (uint32_t r = 0; r < BS_ROUNDS; r++) {
            if (r >= R) break;
            uint32_t j = r * BLK + tid;
            pv[r] = j < len ? __ldg(P + lo + j) : 0u;
        }
#pragma unroll
        for (uint32_t r = 0; r < BS_ROUNDS; r++) {
            if (r >= R) break;
            uint32_t j = r * BLK + tid;
            if (j < len) sk[j] = pv[r];
        }
        __syncthreads();
        for (uint32_t j = tid; j < len; j += BLK) Pout[lo + j] = sk[src[j]];
    }
    if (w == 0) {
        uint32_t prefix = tile_walk_u32(S, tile, (uint32_t)seg_total, tile + 1 == ntiles, d_total);
        if (l == 0) s_prefix = prefix;
    }
    __syncthreads();
    if (!__any_sync(FULL, tb != 0u)) return;                     // warp-uniform: the ballots below need all lanes
    const uint32_t prefix = s_prefix;
    for (uint32_t r = 0; r < R; r++) {
        uint32_t balh = __ballot_sync(FULL, (hb >> r) & 1u), balt = __ballot_sync(FULL, (tb >> r) & 1u);
        if (!((tb >> r) & 1u)) continue;
        const uint32_t j = r * BLK + tid;
        unsigned long long e = s_seg[r * NWARP + w];
        uint32_t le = balh & (lanemask_lt() | (1u << l));
        uint32_t head = le ? r * BLK + w * 32 + 31 - __clz(le) : (uint32_t)(e >> 32);
        uint32_t at = prefix + (uint32_t)e + __popc(balt & lanemask_lt());
        aslot[at] = lo + j;
        apos[at] = Pout[lo + j];
        ahead[at] = lo + head;
    }
}

struct OutMaxInPlace {
    uint32_t *a;
    __device__ void operator()(uint64_t i, uint32_t exc, uint32_t v) const { a[i] = exc > v ? exc : v; }
};

// ---- round r >= 2 over the compacted active list (slot order; groups contiguous)
template <int BITS>
__global__ void __launch_bounds__(BLK) k_lms_refine_keys(LmsWin W, const uint32_t *__restrict__ apos,
                                                         const uint32_t *__restrict__ agrp, uint32_t na, uint32_t h,
                                                         uint64_t *keys) {
    uint32_t j = blockIdx.x * BLK + threadIdx.x;
    if (j >= na) return;
    keys[j] = ((uint64_t)agrp[j] << 32) | lms_window<BITS>(W, apos[j] + h);    // apos + h <= n (not truncated before)
}
struct InLmsGroupR {
    const uint64_t *K; const uint32_t *P, *slot; uint32_t na, n, span;
    __device__ __forceinline__ bool trunc(uint32_t p) const { return (uint64_t)p + span > n; }
    __device__ __forceinline__ bool head(uint32_t j) const {
        return j == 0 || K[j] != K[j - 1] || trunc(P[j - 1]) || trunc(P[j]);
    }
    __device__ unsigned long long operator()(uint64_t jj) const {
        uint32_t j = (uint32_t)jj;
        bool hd = head(j), tl = (j + 1 == na) || head(j + 1);
        return ((unsigned long long)(hd ? slot[j] : 0u) << 32) | ((hd && tl) ? 0u : 1u);
    }
};
struct OutLmsCompactR {
    const uint32_t *P, *slot; uint32_t *list; uint32_t *oslot, *opos, *ogrp;
    __device__ void operator()(uint64_t j, unsigned long long exc, unsigned long long v) const {
        uint32_t p = P[j], sl = slot[j];
        list[sl] = p;                                   // position inside the group is final for this depth
        if ((uint32_t)v) {
            uint32_t eh = (uint32_t)(exc >> 32), vh = (uint32_t)(v >> 32), k = (uint32_t)exc;
            oslot[k] = sl; opos[k] = p; ogrp[k] = eh > vh ? eh : vh;
        }
    }
};

}  // namespace b200sa
