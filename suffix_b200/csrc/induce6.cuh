// induce6.cuh -- K4/K5 for 2-bit packed text (sigma <= 4): the one-round bucket steps of
// induce.cuh (reference src/table.rs:421-448, :543-573, head_insert/tail_insert :723-736) with
//   * PACKED-COUNTER RANKING on physically aligned tiles: tiles are cut in physical index space at
//     multiples of TILE, so thread t owns 8 consecutive, 32-byte aligned entries (two 16-byte
//     loads); the logical (scan) order is thread-major, ascending or descending.  With at most 4
//     destination buckets the per-thread counts of all buckets fit ONE 64-bit word (4 fields of 16
//     bits; a tile has 2048 entries), so one block-wide add-scan of that word ranks the whole tile
//     stably for every bucket at once, and the count matrix of a step is G x 4 words, not G x 256;
//   * 16-bit CARRIED CHARS: a word next to every SA slot holds the next six text chars to the left
//     of the entry, b = c1 | c2 << 2 | ... | c6 << 10 | cnt << 12, written by the step that
//     PRODUCES the entry; a child inherits (b >> 2, cnt - 1) without touching memory, and the
//     producer refreshes a child that would run dry.  Without them the count phases are bound by one
//     divergent T[s-1] gather per entry; with them a count phase reads 2 bytes per entry -- except
//     for LMS lists, whose entries gather once, and the rare entries made by the shared small-step
//     code (marked 0);
//   * CASCADE STEPS for the short chain lists at the end of every bucket (below).
// Control flow (peek, big / small steps, run skipping, fill accounting, invariants) is the one
// of induce.cuh.
#pragma once
#include "induce.cuh"
#ifndef IND6_MINB
#define IND6_MINB 3
#endif

namespace b200sa {

struct Ind6Shared {
    unsigned long long wtot[2][NWARP];   // per-warp packed totals, double buffered over tiles
    uint32_t cbase[4];                   // running destination position per code (inside the bucket part)
    uint32_t sbase[2][4];                // per tile and code: SA slot of staged item 0, double buffered over tiles
    uint32_t ctot[4];                    // step totals per code
    uint32_t code_of[256];
    uint32_t nsig;
};

// Physical chunk of thread t in tile T of a segment: 8 consecutive entries in PHYSICAL order
// (no data movement after the load: the registers are consumed an iteration later, so the
// loads stay in flight under the work on the previous tile).  Logical (scan) order is
// ascending physical index in the L pass and descending in the S pass.
__device__ __forceinline__ void ind6_load8(const uint32_t *__restrict__ src, uint32_t chunk, uint32_t limit,
                                           uint32_t (&raw)[ITEMS]) {
    if (chunk + ITEMS <= limit) {
        const uint4 *q = reinterpret_cast<const uint4 *>(src + chunk);
        uint4 a = __ldcg(q), b = __ldcg(q + 1);
        raw[0] = a.x; raw[1] = a.y; raw[2] = a.z; raw[3] = a.w;
        raw[4] = b.x; raw[5] = b.y; raw[6] = b.z; raw[7] = b.w;
    } else {
#pragma unroll
        for (int i = 0; i < ITEMS; i++) raw[i] = (chunk + i < limit) ? __ldcg(src + chunk + i) : 0u;
    }
}

// pair-reversal of 16 two-bit groups (same as lms_sort.cuh::rev_pairs, which is included later)
__device__ __forceinline__ uint32_t rev_pairs16(uint32_t x) {
    uint32_t y = __brev(x);
    return ((y & 0x55555555u) << 1) | ((y >> 1) & 0x55555555u);
}
// carried word of the entry at text position e from the ONE aligned text word that holds T[e-1]
// (up to six chars; fewer when the word starts within six chars)
__device__ __forceinline__ uint32_t carry_from_word(uint32_t e, uint32_t wd) {
    uint32_t q = e - 1u;                          // position of c1 (e > 0)
    uint32_t av = (q & 15u) + 1u;                 // chars of this word at or below q
    uint32_t x = wd << (2u * (15u - (q & 15u)));  // c1 in the top pair
    uint32_t cnt = av < 6u ? av : 6u;
    return (rev_pairs16(x) & 0xfffu) | (cnt << 12);
}
__device__ __forceinline__ uint32_t fresh_carry(const void *__restrict__ ptext, uint32_t e) {
    if (e == 0) return 0u;
    return carry_from_word(e, __ldg(reinterpret_cast<const uint32_t *>(ptext) + ((e - 1u) >> 4)));
}
// 8 carried words of a lane's chunk (16 bytes)
__device__ __forceinline__ void load_carry8(const uint16_t *__restrict__ pc, uint32_t chunk, uint32_t limit, uint32_t (&v)[4]) {
    if (chunk + ITEMS <= limit) {
        uint4 a = __ldcg(reinterpret_cast<const uint4 *>(pc + chunk));
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    } else {
#pragma unroll
        for (int i = 0; i < 4; i++) {
            uint32_t lo = (chunk + 2 * i < limit) ? pc[chunk + 2 * i] : 0u, hi = (chunk + 2 * i + 1 < limit) ? pc[chunk + 2 * i + 1] : 0u;
            v[i] = lo | (hi << 16);
        }
    }
}
__device__ __forceinline__ uint32_t carry_at(const uint32_t (&v)[4], int i) { return (v[i >> 1] >> ((i & 1) * 16)) & 0xffffu; }

// diagnostics (B200SA_STEPLOG): block 0 logs the phase boundaries of a big step
#define IND_MARK(code)                                                                                   \
    if (A.steplog && bid == 0 && tid == 0) {                                                             \
        unsigned long long now_, k_ = A.steplog[0];                                                      \
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now_));                                         \
        if (k_ < 2000) { A.steplog[1 + 2 * k_] = now_; A.steplog[2 + 2 * k_] = 0xF0000000ull | (code); A.steplog[0] = k_ + 1; } \
    }

// ---------------------------------------------------------------- cascade steps
// The entries a chain list induces into its OWN bucket are the next list of that bucket, a
// quarter as long on random DNA: every bucket ends in a cascade of short steps that each cost two
// grid syncs whatever their size (tools/steplog.py records the step timeline).  With six chars
// carried next to every entry the next CAS_R rounds of an entry are known without touching the
// text: the run r of the bucket char among c1..c5 says that rounds 1..r put s-1..s-r into this
// bucket, and round r+1 puts s-r-1 into bucket c_{r+1} iff that char lies on the valid side (L pass: above, S pass: below;
// the range test is the type test, src/table.rs:430,444).  In the serial scan the products of
// round j+1 follow ALL products of round j in every bucket, in list order, so one step ranks the
// bins (destination, round) -- 4 x CAS_R counters of 12 bits in four 64-bit words, one block-wide
// add-scan -- and leaves the round-CAS_R products as the next list.  Used for chain lists of at
// most one 2048-entry tile per block (grid step) and inside block 0's small episodes.
constexpr int CAS_R = 5;
constexpr unsigned long long CAS_ONES = 0x0001001001001001ull;      // one per 12-bit field

// carried word with min(6, e) chars from the two aligned text words around T[e-1]
__device__ __forceinline__ uint32_t carry_from_words2(uint32_t e, uint32_t hi, uint32_t lo) {
    uint32_t q = e - 1u;
    uint32_t x = __funnelshift_l(lo, hi, 2u * (15u - (q & 15u)));   // c1 in the top pair, c2.. below
    uint32_t cnt = e < 6u ? e : 6u;
    return (rev_pairs16(x) & 0xfffu) | (cnt << 12);
}
__device__ __forceinline__ unsigned long long sel4(uint32_t k, unsigned long long a, unsigned long long b,
                                                   unsigned long long c, unsigned long long d) {
    return k == 0u ? a : k == 1u ? b : k == 2u ? c : d;
}

// One cascade step over the chain list sh.seg of the bucket with byte cbyte.  local: block 0 alone, a
// list of at most TILE entries, no grid sync.  Otherwise every block calls it; block b < tiles owns the
// logical items [b * TILE, (b+1) * TILE).  Leaves fill[] advanced and (st_c, st_phase, st_begin) on the
// products of the last round.  The code is kept SMALL on purpose (rolled loops over a shared-memory copy
// of the tile): it runs a few times per pass, from a cold instruction cache.
template <bool SPASS>
__device__ __noinline__ void cascade_step(const InduceArgs &A, IndShared &sh, Ind6Shared &s4, cg::grid_group &grid,
                                          uint32_t cbyte, uint32_t tiles, uint32_t *cntbuf, bool local) {
    const uint32_t G = gridDim.x, bid = blockIdx.x, tid = threadIdx.x;
    const uint32_t w = warp_id(), l = lane_id();
    const uint32_t Gp = (G + 3u) & ~3u;                 // row stride of the count matrix [4 * CAS_R][Gp]
    const uint32_t cc = s4.code_of[cbyte];
    const uint32_t len = sh.seg.len, base = sh.seg.base;
    uint16_t *pc = reinterpret_cast<uint16_t *>(A.pred);
    unsigned long long *wtot = reinterpret_cast<unsigned long long *>(&sh.wcnt[0][0]);   // [NWARP][4]
    uint32_t *gbase = sh.hist, *tot = sh.tcnt, *bef = sh.base;                            // [4][CAS_R] each
    uint32_t *ent = sh.ent + tid, *car = sh.rl + tid;                 // item i of this thread at [i * BLK]
    const bool active = local || bid < tiles;
    const uint32_t k0 = (local ? 0u : bid * (uint32_t)TILE) + (uint32_t)ITEMS * tid;
    unsigned long long W0 = 0, W1 = 0, W2 = 0, W3 = 0;
    if (active) {
        {
            uint32_t sv[ITEMS], bt[ITEMS], hi[ITEMS], lo[ITEMS];
#pragma unroll
            for (int i = 0; i < ITEMS; i++) {
                uint32_t k = k0 + i;
                uint32_t p = SPASS ? base - k : base + k;
                bool in = k < len;
                sv[i] = in ? __ldcg(A.sa + p) : 0u;
                bt[i] = in ? (uint32_t)__ldcg(pc + p) : 0u;
            }
            // entries with fewer than min(6, s) chars get them now (two aligned words, all loads in flight together)
#pragma unroll
            for (int i = 0; i < ITEMS; i++) {
                uint32_t cnt = bt[i] >> 12;
                bool need = cnt < 6u && cnt < sv[i];
                uint32_t wi = need ? ((sv[i] - 1u) >> 4) : 0u;
                hi[i] = need ? __ldg(reinterpret_cast<const uint32_t *>(A.ptext) + wi) : 0u;
                lo[i] = (need && wi > 0u) ? __ldg(reinterpret_cast<const uint32_t *>(A.ptext) + wi - 1u) : 0u;
            }
#pragma unroll
            for (int i = 0; i < ITEMS; i++) {
                uint32_t cnt = bt[i] >> 12;
                if (cnt < 6u && cnt < sv[i]) bt[i] = carry_from_words2(sv[i], hi[i], lo[i]);
                ent[i * BLK] = sv[i];
                car[i * BLK] = bt[i];
            }
        }
        // ---- count: bins (destination, round) in 12-bit fields
#pragma unroll 1
        for (int i = 0; i < ITEMS; i++) {
            uint32_t b = car[i * BLK];
            uint32_t cnt = b >> 12, ch = b & 0xfffu;
            uint32_t x = ch ^ (cc * 0x555u);
            uint32_t ne = ((x | (x >> 1)) & 0x555u) | (1u << (2u * cnt));
            uint32_t first = (uint32_t)(__ffs(ne) - 1) >> 1;             // leading chars equal to the bucket char (<= cnt)
            uint32_t r = first < (uint32_t)CAS_R ? first : (uint32_t)CAS_R;
            unsigned long long add = CAS_ONES & ((1ull << (12u * r)) - 1ull);
            uint32_t d = cc;
            for (int half = 0; half < 2; half++) {                       // the run (into this bucket), then the terminal
                W0 += d == 0u ? add : 0ull; W1 += d == 1u ? add : 0ull;
                W2 += d == 2u ? add : 0ull; W3 += d == 3u ? add : 0ull;
                d = (ch >> (2u * first)) & 3u;
                bool ok = first < (uint32_t)CAS_R && first < cnt && (SPASS ? d < cc : d > cc);
                add = ok ? (1ull << (12u * first)) : 0ull;
            }
        }
    }
    // ---- block-wide exclusive scan of the four words (threads are in list order)
    unsigned long long I0 = W0, I1 = W1, I2 = W2, I3 = W3;
#pragma unroll 1
    for (int s = 1; s < 32; s <<= 1) {
        unsigned long long t0 = __shfl_up_sync(FULL, I0, s), t1 = __shfl_up_sync(FULL, I1, s);
        unsigned long long t2 = __shfl_up_sync(FULL, I2, s), t3 = __shfl_up_sync(FULL, I3, s);
        if ((int)l >= s) { I0 += t0; I1 += t1; I2 += t2; I3 += t3; }
    }
    __syncthreads();
    if (l == 31) { wtot[w * 4 + 0] = I0; wtot[w * 4 + 1] = I1; wtot[w * 4 + 2] = I2; wtot[w * 4 + 3] = I3; }
    __syncthreads();
    unsigned long long E0 = I0 - W0, E1 = I1 - W1, E2 = I2 - W2, E3 = I3 - W3;
    unsigned long long T0 = 0, T1 = 0, T2 = 0, T3 = 0;
#pragma unroll 1
    for (int ww = 0; ww < NWARP; ww++) {
        unsigned long long a = wtot[ww * 4 + 0], b = wtot[ww * 4 + 1], c = wtot[ww * 4 + 2], d = wtot[ww * 4 + 3];
        if (ww < (int)w) { E0 += a; E1 += b; E2 += c; E3 += d; }
        T0 += a; T1 += b; T2 += c; T3 += d;
    }
    if (tid < 4 * CAS_R) {
        uint32_t d = tid / CAS_R, j = tid % CAS_R;
        uint32_t v = (uint32_t)(sel4(d, T0, T1, T2, T3) >> (12u * j)) & 0xfffu;
        if (local) { tot[tid] = v; bef[tid] = 0u; }
        else if (active) cntbuf[(size_t)tid * Gp + bid] = v;
    }
    if (!local) {
        __syncthreads();
        IND_MARK(1)
        grid.sync();
        IND_MARK(2)
#pragma unroll 1
        for (uint32_t k = w; k < (uint32_t)(4 * CAS_R); k += NWARP) {       // one bin row per warp, four blocks per load
            uint32_t ts = 0, bs = 0;
            for (uint32_t b4 = 4u * l; b4 < tiles; b4 += 128u) {
                uint4 v = __ldcg(reinterpret_cast<const uint4 *>(cntbuf + (size_t)k * Gp + b4));
                uint32_t x0 = v.x, x1 = b4 + 1u < tiles ? v.y : 0u, x2 = b4 + 2u < tiles ? v.z : 0u, x3 = b4 + 3u < tiles ? v.w : 0u;
                ts += x0 + x1 + x2 + x3;
                bs += (b4 < bid ? x0 : 0u) + (b4 + 1u < bid ? x1 : 0u) + (b4 + 2u < bid ? x2 : 0u) + (b4 + 3u < bid ? x3 : 0u);
            }
            ts = __reduce_add_sync(FULL, ts); bs = __reduce_add_sync(FULL, bs);
            if (l == 0) { tot[k] = ts; bef[k] = bs; }
        }
    }
    __syncthreads();
    if (tid < 4) {
        uint32_t run = sh.fill[sh.alpha[tid]];
#pragma unroll 1
        for (int j = 0; j < CAS_R; j++) {
            if (j == CAS_R - 1 && tid == cc) s4.cbase[0] = run;          // where the next list of this bucket begins
            gbase[tid * CAS_R + j] = run + bef[tid * CAS_R + j];
            run += tot[tid * CAS_R + j];
        }
        s4.ctot[tid] = run - sh.fill[sh.alpha[tid]];
    }
    __syncthreads();
    if (!local) { IND_MARK(3) }
    // ---- emit: every entry writes its products of all rounds (SA word + carried word of the child)
    if (active) {
        unsigned long long Ec = sel4(cc, E0, E1, E2, E3);
        const uint32_t bs_c = SPASS ? sh.bstart[cbyte + 1] - 1u : sh.bstart[cbyte];
#pragma unroll 1
        for (int i = 0; i < ITEMS; i++) {
            uint32_t sv = ent[i * BLK], b = car[i * BLK];
            uint32_t cnt = b >> 12, ch = b & 0xfffu;
            uint32_t x = ch ^ (cc * 0x555u);
            uint32_t ne = ((x | (x >> 1)) & 0x555u) | (1u << (2u * cnt));
            uint32_t first = (uint32_t)(__ffs(ne) - 1) >> 1;
            uint32_t r = first < (uint32_t)CAS_R ? first : (uint32_t)CAS_R;
#pragma unroll 1
            for (uint32_t j = 1; j <= r; j++) {
                uint32_t pos = gbase[cc * CAS_R + (j - 1u)] + ((uint32_t)(Ec >> (12u * (j - 1u))) & 0xfffu);
                uint32_t slot = SPASS ? bs_c - pos : bs_c + pos;
                A.sa[slot] = sv - j;
                pc[slot] = (uint16_t)(cnt > j ? ((ch >> (2u * j)) | ((cnt - j) << 12)) : 0u);
            }
            Ec += CAS_ONES & ((1ull << (12u * r)) - 1ull);
            uint32_t d = (ch >> (2u * first)) & 3u;
            if (first < (uint32_t)CAS_R && first < cnt && (SPASS ? d < cc : d > cc)) {
                unsigned long long Ed = sel4(d, E0, E1, E2, E3);
                uint32_t pos = gbase[d * CAS_R + first] + ((uint32_t)(Ed >> (12u * first)) & 0xfffu);
                uint32_t db = sh.alpha[d];
                uint32_t slot = SPASS ? sh.bstart[db + 1] - 1u - pos : sh.bstart[db] + pos;
                uint32_t j = first + 1u;
                A.sa[slot] = sv - j;
                pc[slot] = (uint16_t)(cnt > j ? ((ch >> (2u * j)) | ((cnt - j) << 12)) : 0u);
                unsigned long long one = 1ull << (12u * first);
                E0 += d == 0u ? one : 0ull; E1 += d == 1u ? one : 0ull;
                E2 += d == 2u ? one : 0ull; E3 += d == 3u ? one : 0ull;
            }
        }
    }
    __syncthreads();
    if (tid < 4 && tid < s4.nsig) sh.fill[sh.alpha[tid]] += s4.ctot[tid];
    if (tid == 0) { sh.st_c = (int32_t)cbyte; sh.st_phase = 0; sh.st_begin = s4.cbase[0]; }
    if (!local) {
        IND_MARK(4)
        grid.sync();
    } else __syncthreads();
}

// Small episode of k_induce6: induce_small_episode (induce.cuh) with cascade steps for chain lists.
template <bool SPASS>
__device__ __noinline__ void induce6_small_episode(const InduceArgs &A, IndShared &sh, Ind6Shared &s4, cg::grid_group &grid,
                                                   uint32_t &smallcount) {
    const uint32_t bid = blockIdx.x, tid = threadIdx.x;
    if (bid == 0) {
        while (sh.has && sh.seg.len <= (uint32_t)TILE) {
            Seg g = sh.seg;
            smallcount++;
            const bool chain = sh.is_chain != 0;
            const int32_t cc = sh.ns_c;                 // a chain segment keeps ns_c == its bucket
            __syncthreads();
            if (tid == 0) {
                if (chain && sh.streak_c == cc) sh.streak++;
                else { sh.streak = chain ? 1u : 0u; sh.streak_c = chain ? cc : -1; }
            }
            __syncthreads();
            if (chain && sh.streak >= (A.run_streak ? A.run_streak : RUN_STREAK)) {
                induce_run_skip<SPASS, 2>(A, sh, g, (uint32_t)cc, grid);
                if (tid == 0) { sh.st_c = cc; sh.st_phase = 0; sh.st_begin = sh.fill[cc]; sh.streak = 0; sh.streak_c = -1; }
                __syncthreads();
                if (tid == 0) induce_peek<SPASS>(A, sh);
                __syncthreads();
                continue;
            }
            if (chain && A.cascade) cascade_step<SPASS>(A, sh, s4, grid, (uint32_t)cc, 1u, nullptr, true);
            else {
                sh.base[tid] = sh.fill[tid];
                __syncthreads();
                induce_tile<SPASS, MODE_SMALL, 2>(A, sh, g, 0);
                sh.fill[tid] = sh.base[tid];
                if (tid == 0) { sh.st_c = sh.ns_c; sh.st_phase = sh.ns_phase; sh.st_begin = sh.ns_begin; }
                __syncthreads();
            }
            if (tid == 0) induce_peek<SPASS>(A, sh);
            __syncthreads();
        }
        A.g_fill[tid] = sh.fill[tid];
        if (tid == 0) {
            A.g_state[0] = sh.st_c; A.g_state[1] = sh.st_phase; A.g_state[2] = (int32_t)sh.st_begin;
            A.cmd[0] = CMD_DONE;
        }
        __threadfence();
        grid.sync();
    } else {
        while (true) {
            grid.sync();
            if (__ldcg(A.cmd + 0) != CMD_EMIT) break;
            grid_emit<SPASS>(A, sh);
            grid.sync();
        }
    }
    if (bid != 0) {
        sh.fill[tid] = __ldcg(A.g_fill + tid);
        if (tid == 0) {
            sh.st_c = __ldcg(A.g_state + 0); sh.st_phase = __ldcg(A.g_state + 1);
            sh.st_begin = (uint32_t)__ldcg(A.g_state + 2);
        }
    }
    __syncthreads();
}

// One ordinary (one-round) big step of k_induce6 over sh.seg, all blocks.  A function of its own so that the
// registers of its two tile loops are allocated without regard to the rest of the kernel.
template <bool SPASS>
__device__ __noinline__ void induce6_big_step(const InduceArgs &A, IndShared &sh, Ind6Shared &s4, cg::grid_group &grid,
                                              uint32_t bigcount, uint32_t &bigtiles) {
    const uint32_t G = gridDim.x, bid = blockIdx.x, tid = threadIdx.x;
    const uint32_t w = warp_id(), l = lane_id();
#define BLK_MARK(k)                                                                              \
    if (A.steplog && A.blocklog_step == bigcount + 1u && tid == 0) {                             \
        unsigned long long now_;                                                                 \
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now_));                                 \
        A.steplog[4096 + 6 * bid + (k)] = now_;                                                  \
        if ((k) == 0) { uint32_t sm_; asm volatile("mov.u32 %0, %%smid;" : "=r"(sm_)); A.steplog[4096 + 6 * bid + 5] = sm_; } \
    }
    BLK_MARK(0)
    // -------------------- big step: all blocks
    const Seg &o = sh.seg;
    const uint32_t *src = o.src;
    uint32_t pa, pb;
    if (o.rev) { pb = o.base + 1u; pa = pb - o.len; } else { pa = o.base; pb = o.base + o.len; }
    const uint32_t limit = (o.src == A.sa) ? A.n : sh.S_or_lmsoff[256];
    uint32_t lo = 0, hi = s4.nsig;
    while (lo < s4.nsig && sh.alpha[lo] < o.lo) lo++;
    while (hi > 0 && sh.alpha[hi - 1] > o.hi) hi--;
    const bool gather_all = (src != A.sa);             // LMS list: nothing carried yet
    uint16_t *pc = reinterpret_cast<uint16_t *>(o.pred);         // carried words of this list
    uint16_t *pc_sa = reinterpret_cast<uint16_t *>(A.pred);      // carried words next to the SA slots
    uint32_t *cntbuf = A.blk_cnt + (size_t)(bigcount & 1u) * G * 4u;
    constexpr bool REV = SPASS;
    const uint32_t T0 = pa / TILE, T1 = (pb - 1u) / TILE;
    const uint32_t tiles = T1 - T0 + 1u;
    bigtiles += tiles;
    const uint32_t tpb = (tiles + G - 1) / G;
    const uint32_t nact = (tiles + tpb - 1) / tpb;
    uint32_t tb0 = bid * tpb, tb1 = tb0 + tpb;
    if (tb0 > tiles) tb0 = tiles;
    if (tb1 > tiles) tb1 = tiles;
    auto chunk_of = [&](uint32_t k) -> uint32_t {
        uint32_t T = REV ? (T1 - k) : (T0 + k);
        return REV ? (T * TILE + TILE - 8u * (tid + 1u)) : (T * TILE + 8u * tid);
    };
    // ---- phase A: count
    uint32_t c0 = 0, c1 = 0, c2 = 0, c3 = 0;
    if (gather_all) {
        uint32_t s0[ITEMS], s1[ITEMS], wv[ITEMS];
        if (tb0 < tb1) ind6_load8(src, chunk_of(tb0), limit, s0);
        for (uint32_t k = tb0; k < tb1; k++) {
            if (k + 1 < tb1) ind6_load8(src, chunk_of(k + 1), limit, s1);
            const uint32_t chunk = chunk_of(k);
#pragma unroll
            for (int i = 0; i < ITEMS; i++)           // one aligned text word per entry, all eight in flight
                wv[i] = __ldg(reinterpret_cast<const uint32_t *>(A.ptext) + ((s0[i] > 0 ? s0[i] - 1u : 0u) >> 4));
            uint32_t out[4] = {0, 0, 0, 0};
#pragma unroll
            for (int i = 0; i < ITEMS; i++) {
                uint32_t p = chunk + i;
                bool in = p >= pa && p < pb;
                uint32_t bt = (in && s0[i] > 0) ? carry_from_word(s0[i], wv[i]) : 0u;
                uint32_t d = bt & 3u;
                bool ok = in && (bt >> 12) != 0u && d >= lo && d < hi;
                c0 += (ok && d == 0u); c1 += (ok && d == 1u); c2 += (ok && d == 2u); c3 += (ok && d == 3u);
                out[i >> 1] |= bt << ((i & 1) * 16);
            }
            // neighbours outside the segment belong to other LMS lists, which write theirs when their turn comes
            if (chunk + ITEMS <= limit) *reinterpret_cast<uint4 *>(pc + chunk) = make_uint4(out[0], out[1], out[2], out[3]);
            else {
                for (int i = 0; i < ITEMS; i++) if (chunk + i < limit) pc[chunk + i] = (uint16_t)(out[i >> 1] >> ((i & 1) * 16));
            }
#pragma unroll
            for (int i = 0; i < ITEMS; i++) s0[i] = s1[i];
        }
    } else {
        uint32_t p_cur[4] = {0, 0, 0, 0}, p_nxt[4] = {0, 0, 0, 0};
        if (tb0 < tb1) load_carry8(pc, chunk_of(tb0), limit, p_cur);
        for (uint32_t k = tb0; k < tb1; k++) {
            if (k + 1 < tb1) load_carry8(pc, chunk_of(k + 1), limit, p_nxt);
            const uint32_t chunk = chunk_of(k);
            uint32_t need = 0;
#pragma unroll
            for (int i = 0; i < ITEMS; i++) {
                uint32_t p = chunk + i;
                if (p >= pa && p < pb && (carry_at(p_cur, i) >> 12) == 0u) need |= 1u << i;
            }
            if (need) {                               // products of small steps / the seed: chars not carried
                uint32_t sv[ITEMS];
                ind6_load8(src, chunk, limit, sv);
#pragma unroll
                for (int i = 0; i < ITEMS; i++) {
                    if ((need >> i) & 1u) {
                        uint32_t nb = fresh_carry(A.ptext, sv[i]);
                        p_cur[i >> 1] = (p_cur[i >> 1] & ~(0xffffu << ((i & 1) * 16))) | (nb << ((i & 1) * 16));
                        pc[chunk + i] = (uint16_t)nb;
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < ITEMS; i++) {
                uint32_t p = chunk + i;
                uint32_t bt = carry_at(p_cur, i);
                uint32_t d = bt & 3u;
                bool ok = p >= pa && p < pb && (bt >> 12) != 0u && d >= lo && d < hi;
                c0 += (ok && d == 0u); c1 += (ok && d == 1u); c2 += (ok && d == 2u); c3 += (ok && d == 3u);
            }
#pragma unroll
            for (int i = 0; i < 4; i++) p_cur[i] = p_nxt[i];
        }
    }
    {   // block totals of the 4 codes
        c0 = __reduce_add_sync(FULL, c0); c1 = __reduce_add_sync(FULL, c1);
        c2 = __reduce_add_sync(FULL, c2); c3 = __reduce_add_sync(FULL, c3);
        __syncthreads();
        if (l == 0) { sh.wcnt[w][0] = c0; sh.wcnt[w][1] = c1; sh.wcnt[w][2] = c2; sh.wcnt[w][3] = c3; }
        __syncthreads();
        if (tid < 4 && bid < nact) {
            uint32_t v = 0;
#pragma unroll
            for (int ww = 0; ww < NWARP; ww++) v += sh.wcnt[ww][tid];
            cntbuf[(size_t)bid * 4u + tid] = v;
        }
    }
    __syncthreads();
    IND_MARK(1)
    BLK_MARK(1)
    grid.sync();
    IND_MARK(2)
    BLK_MARK(2)
    // ---- phase B: offsets from the G x 4 count matrix, block-wide stable scatter
    {
        uint32_t be[4] = {0, 0, 0, 0}, to[4] = {0, 0, 0, 0};
        for (uint32_t b = tid; b < nact; b += BLK) {
            uint4 v = __ldcg(reinterpret_cast<const uint4 *>(cntbuf) + b);
            to[0] += v.x; to[1] += v.y; to[2] += v.z; to[3] += v.w;
            if (b < bid) { be[0] += v.x; be[1] += v.y; be[2] += v.z; be[3] += v.w; }
        }
#pragma unroll
        for (int q = 0; q < 4; q++) { be[q] = __reduce_add_sync(FULL, be[q]); to[q] = __reduce_add_sync(FULL, to[q]); }
        if (l == 0) {
#pragma unroll
            for (int q = 0; q < 4; q++) { sh.wcnt[w][8 + q] = be[q]; sh.wcnt[w][12 + q] = to[q]; }
        }
        __syncthreads();
        if (tid < 4) {
            uint32_t bsum = 0, tsum = 0;
#pragma unroll
            for (int ww = 0; ww < NWARP; ww++) { bsum += sh.wcnt[ww][8 + tid]; tsum += sh.wcnt[ww][12 + tid]; }
            s4.cbase[tid] = sh.fill[sh.alpha[tid]] + bsum;
            s4.ctot[tid] = tsum;
        }
    }
    __syncthreads();
    IND_MARK(3)
    if (tb0 < tb1) {
        // the running position of code q lives in s4.cbase[q] (thread q alone advances it); per tile thread
        // q leaves the slot of staged item 0 of its code in s4.sbase, so the store loop keeps no bases in
        // registers
        const uint32_t bsq = tid < 4 ? (SPASS ? sh.bstart[sh.alpha[tid] + 1] - 1u : sh.bstart[sh.alpha[tid]]) : 0u;
        uint32_t s_cur[ITEMS], s_nxt[ITEMS], p_cur[4], p_nxt[4] = {0, 0, 0, 0};
        ind6_load8(src, chunk_of(tb0), limit, s_cur);
        load_carry8(pc, chunk_of(tb0), limit, p_cur);
        uint32_t par = 0;
        for (uint32_t k = tb0; k < tb1; k++) {
            if (k + 1 < tb1) {
                ind6_load8(src, chunk_of(k + 1), limit, s_nxt);
                load_carry8(pc, chunk_of(k + 1), limit, p_nxt);
            }
            const uint32_t chunk = chunk_of(k);
            uint32_t okm = 0, dry = 0;
            unsigned long long mine = 0;
#pragma unroll
            for (int i = 0; i < ITEMS; i++) {
                uint32_t p = chunk + i;
                uint32_t bt = carry_at(p_cur, i);
                uint32_t d = bt & 3u, cnt = bt >> 12;
                bool ok = p >= pa && p < pb && cnt != 0u && d >= lo && d < hi;
                if (ok) { okm |= 1u << i; mine += 1ull << (16 * d); if (cnt == 1u) dry |= 1u << i; }
            }
            // children that would run dry get fresh chars now (every sixth generation of a path);
            // the loads are issued together under the scan, not one per branch
            uint32_t wv[ITEMS];
#pragma unroll
            for (int i = 0; i < ITEMS; i++)
                wv[i] = ((dry >> i) & 1u) && s_cur[i] > 1u ? __ldg(reinterpret_cast<const uint32_t *>(A.ptext) + ((s_cur[i] - 2u) >> 4)) : 0u;
            unsigned long long inc = mine;
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) {
                unsigned long long t = __shfl_up_sync(FULL, inc, s);
                if ((int)l >= s) inc += t;
            }
            if (l == 31) s4.wtot[par][w] = inc;
            __syncthreads();
            unsigned long long wpre = 0, ttot = 0;
#pragma unroll
            for (int ww = 0; ww < NWARP; ww++) {
                unsigned long long t = s4.wtot[par][ww];
                if (ww < (int)w) wpre += t;
                ttot += t;
            }
            unsigned long long exc = wpre + inc - mine;
            // the tile's products are staged in shared memory, bucket-major in output order, and written
            // with consecutive threads on consecutive slots: a direct scatter costs one LSU wavefront per
            // store, and there are two stores per entry here
            const uint32_t t0c = (uint32_t)(ttot & 0xffffu), t1c = (uint32_t)((ttot >> 16) & 0xffffu);
            const uint32_t t2c = (uint32_t)((ttot >> 32) & 0xffffu), t3c = (uint32_t)((ttot >> 48) & 0xffffu);
            const uint32_t o1 = t0c, o2 = t0c + t1c, o3 = o2 + t2c, oall = o3 + t3c;
            uint32_t e0 = (uint32_t)(exc & 0xffffu), e1 = o1 + (uint32_t)((exc >> 16) & 0xffffu);
            uint32_t e2 = o2 + (uint32_t)((exc >> 32) & 0xffffu), e3 = o3 + (uint32_t)((exc >> 48) & 0xffffu);
            if (tid < 4) {      // item j of code q (staged at o_q + i) goes to position cbase[q] + i
                const uint32_t oq = tid == 0 ? 0u : tid == 1 ? o1 : tid == 2 ? o2 : o3;
                const uint32_t rb = s4.cbase[tid];
                s4.sbase[par][tid] = SPASS ? bsq - rb + oq : bsq + rb - oq;
                s4.cbase[tid] = rb + (uint32_t)((ttot >> (16 * tid)) & 0xffffu);
            }
            uint16_t *stage_c = reinterpret_cast<uint16_t *>(sh.rl);
#pragma unroll
            for (int ii = 0; ii < ITEMS; ii++) {
                const int i = REV ? (ITEMS - 1 - ii) : ii;           // logical order inside the chunk
                if ((okm >> i) & 1u) {
                    uint32_t bt = carry_at(p_cur, i);
                    uint32_t d = bt & 3u, cnt = bt >> 12;
                    uint32_t cb;
                    if (cnt >= 2u) cb = ((bt >> 2) & 0x3ffu) | ((cnt - 1u) << 12);
                    else cb = (s_cur[i] > 1u) ? carry_from_word(s_cur[i] - 1u, wv[i]) : 0u;
                    uint32_t at = (d == 0u) ? e0++ : (d == 1u) ? e1++ : (d == 2u) ? e2++ : e3++;
                    sh.ent[at] = s_cur[i] - 1u;
                    stage_c[at] = (uint16_t)cb;
                }
            }
            __syncthreads();
            for (uint32_t j = tid; j < oall; j += BLK) {
                const uint32_t q = (j >= o1) + (j >= o2) + (j >= o3);
                const uint32_t sb = s4.sbase[par][q];
                uint32_t slot = SPASS ? sb - j : sb + j;
                A.sa[slot] = sh.ent[j];
                pc_sa[slot] = stage_c[j];
            }
            par ^= 1u;
#pragma unroll
            for (int i = 0; i < ITEMS; i++) s_cur[i] = s_nxt[i];
#pragma unroll
            for (int i = 0; i < 4; i++) p_cur[i] = p_nxt[i];
        }
    }
    __syncthreads();
    if (tid < 4 && tid < s4.nsig) sh.fill[sh.alpha[tid]] += s4.ctot[tid];
    if (tid == 0) { sh.st_c = sh.ns_c; sh.st_phase = sh.ns_phase; sh.st_begin = sh.ns_begin; }
    IND_MARK(4)
    BLK_MARK(3)
    grid.sync();
    BLK_MARK(4)
#undef BLK_MARK
}

template <bool SPASS>
__global__ void __launch_bounds__(BLK, IND6_MINB) k_induce6(InduceArgs A) {
    __shared__ IndShared sh;
    __shared__ Ind6Shared s4;
    cg::grid_group grid = cg::this_grid();
    const uint32_t G = gridDim.x, bid = blockIdx.x, tid = threadIdx.x;
    const uint32_t w = warp_id(), l = lane_id();

    // ---- init: tables, fill counters, seed (suffix n-1 is L: src/table.rs:422-425)
    sh.bstart[tid] = A.bstart[tid];
    if (tid == 0) sh.bstart[256] = A.bstart[256];
    sh.Lcnt[tid] = A.Lcnt[tid];
    if (SPASS) sh.S_or_lmsoff[tid] = A.Scnt[tid];
    else { sh.S_or_lmsoff[tid] = A.lms_off[tid]; if (tid == 0) sh.S_or_lmsoff[256] = A.lms_off[256]; }
    if (tid < 16) sh.alpha[tid] = A.alpha[tid];
    uint32_t lastc = A.text[A.n - 1];
    sh.fill[tid] = (!SPASS && tid == lastc) ? 1u : 0u;
    if (tid == 0) { sh.st_c = SPASS ? 255 : 0; sh.st_phase = 0; sh.st_begin = 0; sh.streak = 0; sh.streak_c = -1; }
    {
        uint32_t present = (A.Lcnt[tid] + A.Scnt[tid]) > 0 ? 1u : 0u, total;
        uint32_t inc = block_incl_scan<OpSum>(present, sh.sw, &total);
        s4.code_of[tid] = inc - present;
        if (tid == 0) s4.nsig = total;
    }
    __syncthreads();
    if (!SPASS && bid == 0 && tid == 0) { A.sa[sh.bstart[lastc]] = A.n - 1u; reinterpret_cast<uint16_t *>(A.pred)[sh.bstart[lastc]] = 0; }
    uint32_t bigcount = 0, smallcount = 0, bigtiles = 0;

    while (true) {
        if (tid == 0) induce_peek<SPASS>(A, sh);
        __syncthreads();
        if (A.steplog && bid == 0 && tid == 0) {
            unsigned long long now, k = A.steplog[0];
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (k < 2000) { A.steplog[1 + 2 * k] = now; A.steplog[2 + 2 * k] = sh.has ? sh.seg.len : 0u; A.steplog[0] = k + 1; }
        }
        if (!sh.has) break;
        if (sh.seg.len <= (uint32_t)TILE) {
            induce6_small_episode<SPASS>(A, sh, s4, grid, smallcount);
            continue;
        }
        if (A.cascade && sh.is_chain && sh.seg.len <= A.cascade) {        // at most one tile per block: all rounds at once
            const uint32_t tiles = (sh.seg.len + TILE - 1) / TILE;
            bigtiles += tiles;
            cascade_step<SPASS>(A, sh, s4, grid, (uint32_t)sh.ns_c, tiles,
                                A.blk_cnt + (size_t)G * 8u + (size_t)(bigcount & 1u) * G * 32u, false);
            bigcount++;
            continue;
        }
        induce6_big_step<SPASS>(A, sh, s4, grid, bigcount, bigtiles);
        bigcount++;
    }
    if (bid == 0 && tid == 0) {
        A.err[4 + (SPASS ? 3 : 0)] = bigcount; A.err[5 + (SPASS ? 3 : 0)] = smallcount; A.err[6 + (SPASS ? 3 : 0)] = bigtiles;
    }
}

}  // namespace b200sa
