// induce.cuh -- K4/K5: the L-then-S induced fill as ONE persistent cooperative
// kernel per pass.  Replaces the four serial induce loops of the reference
// (src/table.rs:421-448 and :543-573) together with Bins::head_insert /
// tail_insert (src/table.rs:723-736).
//
// Parallel formulation (validated on CPU by tests/model_pipeline.py):
//   * buckets are visited in scan order (ascending for L, descending for S);
//   * inside bucket c the serial scan is a sequence of *lists*: the entries
//     already present (induced from earlier buckets), then the entries those
//     induce into c itself (chain round 1), then round 2, ... and finally the
//     second list (L pass: the LMS suffixes of c; S pass: the L part of c);
//   * every list is one stable multi-way partition step by d = T[s-1]:
//     entry s emits s-1 into bucket d iff d is in the list's valid range
//     (no type lookups are needed: the range encodes the type test).
//   A step is either "big" (all blocks: count -> grid.sync -> scatter ->
//   grid.sync) or "small" (<= TILE entries: block 0 alone, no grid sync; it
//   keeps consuming small steps and then hands its state to the grid).
// The per-bucket fill counters (the reference's bin pointers) live in shared
// memory of every block and are advanced identically by all blocks.
#pragma once
#include <cooperative_groups.h>
#include "common.cuh"
#include "classify.cuh"

namespace b200sa {
namespace cg = cooperative_groups;

struct InduceArgs {
    const uint8_t *text;     // level-0 text (bytes)
    const void *ptext;       // packed text (BITS 2/4) or the bytes themselves (BITS 8)
    const uint32_t *alpha;   // code -> byte (BITS < 8)
    uint32_t n;
    uint32_t *sa;            // n slots
    uint8_t *pred;           // n bytes: T[s-1] of the entry in SA slot p (big steps only)
    const uint32_t *lms;     // LMS suffixes grouped by first byte (m)
    uint8_t *lms_pred;       // m bytes
    const uint32_t *bstart;  // [257]
    const uint32_t *Lcnt;    // [256]
    const uint32_t *Scnt;    // [256]
    const uint32_t *lms_off; // [257]
    uint32_t *blk_cnt;       // [2][gridDim.x][256]
    uint32_t *g_fill;        // [256] hand-off after small episodes
    int32_t *g_state;        // [4]   hand-off: c, phase, begin
    uint32_t *err;           // [4]   err[0] != 0 => invariant violated
    uint32_t *run_scratch;   // [TILE] run-skipping: terminal entries in scan order
    uint32_t *run_alive;     // [TILE] run-skipping: alive entries of the epoch being emitted grid-wide
    uint32_t *cmd;           // [8]    block 0 -> grid: {cmd, a, t_prev, rounds, base pos, bucket}
    int carry;               // 2: pred[] carries predecessor chars per SA slot as 16-bit words (k_induce6); products of
                             // the shared small-step code mark theirs "unknown" (0).  0: k_induce
    uint32_t cascade;        // k_induce6: chain lists of at most this many entries take cascade steps (0: off)
    uint32_t run_streak;     // small chain rounds in one bucket before the chain is finished at once (0: RUN_STREAK)
    uint32_t blocklog_step;  // diagnostics: every block logs its phase times of big step number blocklog_step-1 at steplog[4096 + 6*bid ..]
    unsigned long long *steplog;   // diagnostics (B200SA_STEPLOG): [0] = count, then (globaltimer ns, list length) pairs
};
enum { CMD_NONE = 0, CMD_EMIT = 1, CMD_DONE = 2 };
constexpr uint64_t EMIT_GRID_MIN = 32768;   // epochs with at least this many entries are emitted by the whole grid

struct Seg {
    const uint32_t *src;
    uint8_t *pred;
    uint32_t base;   // physical index of logical item 0
    uint32_t len;
    uint32_t lo, hi; // valid destination range (inclusive)
    int rev;         // logical k -> physical base - k
};

struct IndShared {
    uint32_t bstart[257];
    uint32_t Lcnt[256];
    uint32_t S_or_lmsoff[257];   // L pass: lms_off; S pass: Scnt
    uint32_t fill[256];
    uint32_t base[256];
    uint32_t hist[256];
    uint32_t tcnt[256];
    uint32_t wcnt[NWARP][256];
    uint32_t alpha[16];
    // run skipping (block 0, small episodes)
    uint32_t ent[TILE];      // entries of the current chain list
    uint32_t rl[TILE];       // their run lengths to the left
    uint32_t alive[TILE];    // entries still alive in the current epoch, in list order
    uint32_t sw[NWARP + 1];
    uint32_t red;
    uint32_t streak;
    int32_t streak_c;
    int32_t is_chain;
    // broadcast area
    int32_t st_c, st_phase;
    uint32_t st_begin;
    int32_t ns_c, ns_phase;
    uint32_t ns_begin;
    int32_t has;
    Seg seg;
};

enum { MODE_COUNT = 0, MODE_SCATTER = 1, MODE_SMALL = 2 };

// ---- tile pieces.  A tile is the logical items [t0, t0+TILE) ∩ [0, g.len) of
// segment g in the warp-blocked layout of tile_rank.  The big-step loops below
// prefetch the next tile's loads before working on the current one.
__device__ __forceinline__ void tile_load_s(const Seg &g, uint32_t t0, uint32_t (&s)[ITEMS]) {
    const uint32_t w = warp_id(), l = lane_id();
#pragma unroll
    for (int r = 0; r < ITEMS; r++) {
        uint32_t k = t0 + w * (ITEMS * 32) + r * 32 + l;
        uint32_t p = g.rev ? g.base - k : g.base + k;
        s[r] = (k < g.len) ? __ldcg(g.src + p) : 0u;
    }
}
__device__ __forceinline__ void tile_load_pred(const Seg &g, uint32_t t0, uint32_t (&d)[ITEMS]) {
    const uint32_t w = warp_id(), l = lane_id();
#pragma unroll
    for (int r = 0; r < ITEMS; r++) {
        uint32_t k = t0 + w * (ITEMS * 32) + r * 32 + l;
        uint32_t p = g.rev ? g.base - k : g.base + k;
        d[r] = (k < g.len) ? (uint32_t)__ldcg(g.pred + p) : 0u;
    }
}
template <int BITS>
__device__ __forceinline__ void tile_gather(const InduceArgs &A, const IndShared &sh, const uint32_t (&s)[ITEMS],
                                            uint32_t (&d)[ITEMS]) {
#pragma unroll
    for (int r = 0; r < ITEMS; r++) {
        if (BITS == 8) d[r] = (s[r] > 0) ? text_get<8>(A.ptext, s[r] - 1) : 0u;
        else d[r] = (s[r] > 0) ? sh.alpha[text_get<BITS>(A.ptext, s[r] - 1)] : 0u;
    }
}
__device__ __forceinline__ uint32_t tile_valid(const Seg &g, uint32_t t0, const uint32_t (&s)[ITEMS],
                                               const uint32_t (&d)[ITEMS]) {
    const uint32_t w = warp_id(), l = lane_id();
    uint32_t vm = 0;
#pragma unroll
    for (int r = 0; r < ITEMS; r++) {
        uint32_t k = t0 + w * (ITEMS * 32) + r * 32 + l;
        bool valid = k < g.len && s[r] > 0 && d[r] >= g.lo && d[r] <= g.hi;
        vm |= (valid ? 1u : 0u) << r;
    }
    return vm;
}
// count phase of a big step: remember T[s-1] per slot, histogram the valid ones
__device__ __forceinline__ void tile_count(IndShared &sh, const Seg &g, uint32_t t0, const uint32_t (&s)[ITEMS],
                                           const uint32_t (&d)[ITEMS]) {
    const uint32_t w = warp_id(), l = lane_id();
    uint32_t vm = tile_valid(g, t0, s, d);
#pragma unroll
    for (int r = 0; r < ITEMS; r++) {
        uint32_t k = t0 + w * (ITEMS * 32) + r * 32 + l;
        uint32_t p = g.rev ? g.base - k : g.base + k;
        if (k < g.len) g.pred[p] = (uint8_t)d[r];
        hist_add_private(sh.wcnt[w], d[r], (vm >> r) & 1u);     // per-warp private counters
    }
}
// stable scatter of one tile (s, d given); advances sh.base by the tile's counts
template <bool SPASS>
__device__ __forceinline__ void tile_scatter(const InduceArgs &A, IndShared &sh, const Seg &g, uint32_t t0,
                                             const uint32_t (&s)[ITEMS], const uint32_t (&d)[ITEMS]) {
    const uint32_t w = warp_id();
    uint32_t rank[ITEMS];
#pragma unroll
    for (int ww = 0; ww < NWARP; ww++) sh.wcnt[ww][threadIdx.x] = 0;
    __syncthreads();
    uint32_t vm = tile_valid(g, t0, s, d);
    tile_rank(d, vm, rank, sh.wcnt, sh.tcnt);
#pragma unroll
    for (int r = 0; r < ITEMS; r++) {
        if ((vm >> r) & 1u) {
            uint32_t pos = sh.base[d[r]] + sh.wcnt[w][d[r]] + rank[r];
            uint32_t slot = SPASS ? (sh.bstart[d[r] + 1] - 1u - pos) : (sh.bstart[d[r]] + pos);
            A.sa[slot] = s[r] - 1u;
            if (A.carry == 1) A.pred[slot] = 0; else if (A.carry == 2) reinterpret_cast<uint16_t *>(A.pred)[slot] = 0;
        }
    }
    __syncthreads();
    sh.base[threadIdx.x] += sh.tcnt[threadIdx.x];
    __syncthreads();
}
// one whole tile in a small step (block 0): load, gather, scatter
template <bool SPASS, int MODE, int BITS>
__device__ __forceinline__ void induce_tile(const InduceArgs &A, IndShared &sh, const Seg &g, uint32_t t0) {
    uint32_t s[ITEMS], d[ITEMS];
    tile_load_s(g, t0, s);
    tile_gather<BITS>(A, sh, s, d);
    tile_scatter<SPASS>(A, sh, g, t0, s, d);
}

// Thread 0: derive the next non-empty segment from (state, fill) without
// consuming it; ns_* is the state to adopt once it has been processed.
template <bool SPASS>
__device__ void induce_peek(const InduceArgs &A, IndShared &sh) {
    int32_t c = sh.st_c, phase = sh.st_phase;
    uint32_t begin = sh.st_begin;
    sh.has = 0;
    sh.is_chain = 0;
    while (SPASS ? (c >= 0) : (c <= 255)) {
        if (phase == 0) {
            uint32_t end = sh.fill[c];
            if (end > begin) {
                sh.seg.src = A.sa; sh.seg.pred = A.pred; sh.seg.len = end - begin;
                if (SPASS) { sh.seg.base = sh.bstart[c + 1] - 1u - begin; sh.seg.lo = 0; sh.seg.hi = (uint32_t)c; sh.seg.rev = 1; }
                else       { sh.seg.base = sh.bstart[c] + begin; sh.seg.lo = (uint32_t)c; sh.seg.hi = 255; sh.seg.rev = 0; }
                sh.ns_c = c; sh.ns_phase = 0; sh.ns_begin = end; sh.has = 1; sh.is_chain = 1;
                return;
            }
            // chain exhausted: the part must be complete (reference invariant)
            uint32_t want = SPASS ? sh.S_or_lmsoff[c] : sh.Lcnt[c];
            if (end != want && blockIdx.x == 0) { A.err[0] = 1; A.err[1] = (uint32_t)c; A.err[2] = end; A.err[3] = want; }
            phase = 1;
        }
        if (SPASS) {
            uint32_t L = sh.Lcnt[c];
            int32_t cc = c;
            c = c - 1; phase = 0; begin = 0;
            if (L > 0 && cc > 0) {
                sh.seg.src = A.sa; sh.seg.pred = A.pred; sh.seg.len = L;
                sh.seg.base = sh.bstart[cc] + L - 1u; sh.seg.lo = 0; sh.seg.hi = (uint32_t)(cc - 1); sh.seg.rev = 1;
                sh.ns_c = c; sh.ns_phase = 0; sh.ns_begin = 0; sh.has = 1;
                return;
            }
        } else {
            uint32_t a = sh.S_or_lmsoff[c], b = sh.S_or_lmsoff[c + 1];
            int32_t cc = c;
            c = c + 1; phase = 0; begin = 0;
            if (b > a && cc < 255) {
                sh.seg.src = A.lms; sh.seg.pred = A.lms_pred; sh.seg.len = b - a;
                sh.seg.base = a; sh.seg.lo = (uint32_t)(cc + 1); sh.seg.hi = 255; sh.seg.rev = 0;
                sh.ns_c = c; sh.ns_phase = 0; sh.ns_begin = 0; sh.has = 1;
                return;
            }
        }
    }
    sh.st_c = c; sh.st_phase = 0; sh.st_begin = 0;   // done
}

// ---------------------------------------------------------------- run skipping
// A chain inside bucket c advances one position per round along a run of the
// byte c, so a run of length 10^7 (poly-N in a genome, zero padding) would cost
// 10^7 rounds.  Once a bucket has needed RUN_STREAK consecutive small chain
// rounds, block 0 finishes the whole chain of the bucket at once: with l_j the
// length of the run of c to the left of entry e_j of the current list, round r
// emits {e_j - r : l_j >= r} in list order.  Rounds between two consecutive
// distinct l values share one alive set ("epoch"), so each epoch is one block
// scan plus a fully parallel emission.  The entries that end their run
// ("terminals", e_j - l_j, in (l_j, j) order = their order in SA) are then
// pushed through one ordinary small step for the other buckets.
constexpr uint32_t RUN_STREAK = 8;
constexpr uint32_t RUN_LOCAL = 64;          // per-thread probe before the cooperative scan
constexpr uint32_t RUN_INF = 0xffffffffu;

// number of consecutive bytes == c at positions start, start-1, ... (block-cooperative)
__device__ __noinline__ uint32_t run_left_coop(const uint8_t *__restrict__ text, uint32_t start, uint32_t c, IndShared &sh) {
    uint32_t count = 0;
    int64_t cur = start;
    while (true) {
        if (threadIdx.x == 0) sh.red = RUN_INF;
        __syncthreads();
        uint32_t first = RUN_INF;
        for (int q = 0; q < 16; q++) {
            int64_t pos = cur - ((int64_t)threadIdx.x * 16 + q);
            bool same = pos >= 0 && (uint32_t)__ldg(text + pos) == c;
            if (!same) { first = threadIdx.x * 16 + q; break; }
        }
        if (first != RUN_INF) atomicMin(&sh.red, first);
        __syncthreads();
        uint32_t m = sh.red;
        __syncthreads();
        if (m != RUN_INF) return count + m;
        count += 4096;
        cur -= 4096;
    }
}

// Emission share of one block for an epoch published in A.cmd (all blocks call it
// between two grid syncs): rounds t_prev+1 .. t_prev+rounds, `a` alive entries each.
template <bool SPASS>
__device__ __forceinline__ void grid_emit(const InduceArgs &A, const IndShared &sh) {
    const uint32_t a = __ldcg(A.cmd + 1), t_prev = __ldcg(A.cmd + 2), rounds = __ldcg(A.cmd + 3);
    const uint32_t basepos = __ldcg(A.cmd + 4), c = __ldcg(A.cmd + 5);
    const uint64_t items = (uint64_t)rounds * a;
    for (uint64_t idx = (uint64_t)blockIdx.x * BLK + threadIdx.x; idx < items; idx += (uint64_t)gridDim.x * BLK) {
        uint32_t r_off = (uint32_t)(idx / a), jj = (uint32_t)(idx % a);
        uint32_t pos = basepos + (uint32_t)idx;
        uint32_t slot = SPASS ? (sh.bstart[c + 1] - 1u - pos) : (sh.bstart[c] + pos);
        A.sa[slot] = __ldcg(A.run_alive + jj) - (t_prev + 1u + r_off);
        if (A.carry == 1) A.pred[slot] = 0; else if (A.carry == 2) reinterpret_cast<uint16_t *>(A.pred)[slot] = 0;
    }
}

template <bool SPASS, int BITS>
__device__ __noinline__ void induce_run_skip(const InduceArgs &A, IndShared &sh, const Seg &g, uint32_t c,
                                             cg::grid_group &grid) {
    const uint32_t tid = threadIdx.x;
    const uint32_t k = g.len;                       // <= TILE; thread t owns list items [8t, 8t+8)
    // ---- entries and locally probed run lengths
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
        uint32_t j = tid * ITEMS + i;
        uint32_t e = 0, r = 0;
        if (j < k) {
            uint32_t p = g.rev ? g.base - j : g.base + j;
            e = __ldcg(g.src + p);
            while (r < RUN_LOCAL && e > r && (uint32_t)__ldg(A.text + (e - 1 - r)) == c) r++;
            if (r == RUN_LOCAL) r = RUN_INF;        // long: resolved cooperatively below
        }
        sh.ent[j] = e;
        sh.rl[j] = r;
    }
    __syncthreads();
    for (uint32_t j = 0; j < k; j++) {
        if (sh.rl[j] == RUN_INF) {                  // uniform across the block
            uint32_t e = sh.ent[j];
            uint32_t more = (e > RUN_LOCAL) ? run_left_coop(A.text, e - 1 - RUN_LOCAL, c, sh) : 0u;
            __syncthreads();
            if (tid == 0) sh.rl[j] = RUN_LOCAL + more;
            __syncthreads();
        }
    }
    const uint32_t F = sh.fill[c];
    uint64_t O = 0;                                 // chain entries emitted so far
    uint32_t tcount = 0;                            // terminals emitted so far
    uint32_t t_prev = 0;
    bool first_epoch = true;                        // epoch 0 only collects the terminals with l == 0
    while (true) {
        // threshold of this epoch: smallest run length > t_prev (or, first, exactly 0)
        uint32_t thr;
        if (first_epoch) thr = 0;
        else {
            uint32_t mine = RUN_INF;
#pragma unroll
            for (int i = 0; i < ITEMS; i++) {
                uint32_t j = tid * ITEMS + i;
                if (j < k && sh.rl[j] > t_prev && sh.rl[j] < mine) mine = sh.rl[j];
            }
            if (tid == 0) sh.red = RUN_INF;
            __syncthreads();
            if (mine != RUN_INF) atomicMin(&sh.red, mine);
            __syncthreads();
            thr = sh.red;
            __syncthreads();
            if (thr == RUN_INF) break;
            // alive set of rounds t_prev+1 .. thr: run length >= thr
            uint32_t own = 0;
#pragma unroll
            for (int i = 0; i < ITEMS; i++) {
                uint32_t j = tid * ITEMS + i;
                if (j < k && sh.rl[j] >= thr) own++;
            }
            uint32_t a;
            uint32_t inc = block_incl_scan<OpSum>(own, sh.sw, &a);
            uint32_t at = inc - own;
#pragma unroll
            for (int i = 0; i < ITEMS; i++) {
                uint32_t j = tid * ITEMS + i;
                if (j < k && sh.rl[j] >= thr) sh.alive[at++] = sh.ent[j];
            }
            __syncthreads();
            uint64_t items = (uint64_t)(thr - t_prev) * a;
            if (items >= EMIT_GRID_MIN) {
                // big epoch (long runs): publish it and let the whole grid emit
                for (uint32_t q = tid; q < a; q += BLK) A.run_alive[q] = sh.alive[q];
                if (tid == 0) {
                    A.cmd[1] = a; A.cmd[2] = t_prev; A.cmd[3] = thr - t_prev; A.cmd[4] = F + (uint32_t)O; A.cmd[5] = c;
                    A.cmd[0] = CMD_EMIT;
                }
                __threadfence();
                grid.sync();
                grid_emit<SPASS>(A, sh);
                grid.sync();
            } else {
                for (uint64_t idx = tid; idx < items; idx += BLK) {
                    uint32_t r_off = (uint32_t)(idx / a), jj = (uint32_t)(idx % a);
                    uint32_t pos = F + (uint32_t)(O + idx);
                    uint32_t slot = SPASS ? (sh.bstart[c + 1] - 1u - pos) : (sh.bstart[c] + pos);
                    A.sa[slot] = sh.alive[jj] - (t_prev + 1u + r_off);
                    if (A.carry == 1) A.pred[slot] = 0; else if (A.carry == 2) reinterpret_cast<uint16_t *>(A.pred)[slot] = 0;
                }
            }
            O += items;
        }
        // terminals of this epoch: run length == thr, in list order
        {
            uint32_t own = 0;
#pragma unroll
            for (int i = 0; i < ITEMS; i++) {
                uint32_t j = tid * ITEMS + i;
                if (j < k && sh.rl[j] == thr) own++;
            }
            uint32_t tot;
            uint32_t inc = block_incl_scan<OpSum>(own, sh.sw, &tot);
            uint32_t at = tcount + inc - own;
#pragma unroll
            for (int i = 0; i < ITEMS; i++) {
                uint32_t j = tid * ITEMS + i;
                if (j < k && sh.rl[j] == thr) A.run_scratch[at++] = sh.ent[j] - thr;
            }
            tcount += tot;
            __syncthreads();
        }
        t_prev = thr;
        first_epoch = false;
    }
    __syncthreads();
    if (tid == c) sh.fill[c] = F + (uint32_t)O;
    __syncthreads();
    // ---- the terminals feed the other buckets through one ordinary small step
    Seg ts;
    ts.src = A.run_scratch; ts.pred = nullptr; ts.base = 0; ts.len = tcount; ts.rev = 0;
    if (SPASS) { ts.lo = (c > 0) ? 0u : 1u; ts.hi = (c > 0) ? c - 1u : 0u; }
    else       { ts.lo = c + 1u; ts.hi = 255u; }
    sh.base[tid] = sh.fill[tid];
    __syncthreads();
    induce_tile<SPASS, MODE_SMALL, BITS>(A, sh, ts, 0);
    sh.fill[tid] = sh.base[tid];
    __syncthreads();
}

// ---------------- small episode: block 0 alone consumes consecutive small steps (lists of at
// most TILE entries, one chain round per step, run skipping for long runs) and then hands
// its fill counters / state to the grid; the other blocks serve grid-wide emission
// requests of the run skipping while they wait.  All blocks call this with sh.has set
// and sh.seg.len <= TILE.
template <bool SPASS, int BITS>
__device__ __noinline__ void induce_small_episode(const InduceArgs &A, IndShared &sh, cg::grid_group &grid,
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
                induce_run_skip<SPASS, BITS>(A, sh, g, (uint32_t)cc, grid);
                if (tid == 0) { sh.st_c = cc; sh.st_phase = 0; sh.st_begin = sh.fill[cc]; sh.streak = 0; sh.streak_c = -1; }
                __syncthreads();
                if (tid == 0) induce_peek<SPASS>(A, sh);
                __syncthreads();
                continue;
            }
            sh.base[tid] = sh.fill[tid];
            __syncthreads();
            induce_tile<SPASS, MODE_SMALL, BITS>(A, sh, g, 0);
            sh.fill[tid] = sh.base[tid];
            if (tid == 0) { sh.st_c = sh.ns_c; sh.st_phase = sh.ns_phase; sh.st_begin = sh.ns_begin; }
            __syncthreads();
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
        // wait for block 0; serve grid-wide emission requests of its run skipping meanwhile
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

#ifndef INDUCE_MINB
#define INDUCE_MINB 2
#endif
template <bool SPASS, int BITS>
__global__ void __launch_bounds__(BLK, INDUCE_MINB) k_induce(InduceArgs A) {
    __shared__ IndShared sh;
    cg::grid_group grid = cg::this_grid();
    const uint32_t G = gridDim.x, bid = blockIdx.x, tid = threadIdx.x;

    // ---- init: tables, fill counters, seed (suffix n-1 is L: src/table.rs:422-425)
    sh.bstart[tid] = A.bstart[tid];
    if (tid == 0) sh.bstart[256] = A.bstart[256];
    sh.Lcnt[tid] = A.Lcnt[tid];
    if (SPASS) sh.S_or_lmsoff[tid] = A.Scnt[tid];
    else { sh.S_or_lmsoff[tid] = A.lms_off[tid]; if (tid == 0) sh.S_or_lmsoff[256] = A.lms_off[256]; }
    if (BITS < 8 && tid < 16) sh.alpha[tid] = A.alpha[tid];
    uint32_t lastc = A.text[A.n - 1];
    sh.fill[tid] = (!SPASS && tid == lastc) ? 1u : 0u;
    if (tid == 0) { sh.st_c = SPASS ? 255 : 0; sh.st_phase = 0; sh.st_begin = 0; sh.streak = 0; sh.streak_c = -1; }
    __syncthreads();
    if (!SPASS && bid == 0 && tid == 0) A.sa[sh.bstart[lastc]] = A.n - 1u;
    uint32_t bigcount = 0, smallcount = 0, bigtiles = 0;

    while (true) {
        if (tid == 0) induce_peek<SPASS>(A, sh);
        __syncthreads();
        if (!sh.has) break;
        if (sh.seg.len <= (uint32_t)TILE) {
            induce_small_episode<SPASS, BITS>(A, sh, grid, smallcount);
            continue;
        }
        // -------------------- big step: all blocks
        Seg g = sh.seg;
        uint32_t *cntbuf = A.blk_cnt + (size_t)(bigcount & 1u) * G * 256u;
        bigcount++;
        uint32_t tiles = (g.len + TILE - 1) / TILE;
        bigtiles += tiles;
        uint32_t tpb = (tiles + G - 1) / G;
        uint32_t nact = (tiles + tpb - 1) / tpb;
        uint32_t tb0 = bid * tpb, tb1 = tb0 + tpb;
        if (tb1 > tiles) tb1 = tiles;
        // phase A: count + remember predecessors
#pragma unroll
        for (int ww = 0; ww < NWARP; ww++) sh.wcnt[ww][tid] = 0;
        __syncthreads();
        if (tb0 < tb1) {
            uint32_t s_cur[ITEMS], s_nxt[ITEMS], d_cur[ITEMS];
            tile_load_s(g, tb0 * TILE, s_cur);
            for (uint32_t t = tb0; t < tb1; t++) {
                if (t + 1 < tb1) tile_load_s(g, (t + 1) * TILE, s_nxt);      // prefetch under the gather
                tile_gather<BITS>(A, sh, s_cur, d_cur);
                tile_count(sh, g, t * TILE, s_cur, d_cur);
#pragma unroll
                for (int r = 0; r < ITEMS; r++) s_cur[r] = s_nxt[r];
            }
        }
        __syncthreads();
        if (bid < nact) {
            uint32_t v = 0;
#pragma unroll
            for (int ww = 0; ww < NWARP; ww++) v += sh.wcnt[ww][tid];
            cntbuf[(size_t)bid * 256u + tid] = v;
        }
        __syncthreads();      // wcnt is reused by the scatter phase
        grid.sync();
        // phase B: offsets, scatter
        {
            // column sums of the nact x 256 count matrix: rows are dealt to the warps and every lane
            // reads 8 columns of a row with two 16-byte loads, so the whole matrix is in flight at once
            // (one thread per column walking nact rows cost ~nact/4 L2 round trips per step: the largest
            // fixed cost of the ~1000 steps of a sigma = 256 pass)
            uint32_t bacc[8], tacc[8];
#pragma unroll
            for (int j = 0; j < 8; j++) { bacc[j] = 0; tacc[j] = 0; }
            const uint32_t wq = warp_id(), lq = lane_id();
#pragma unroll 4
            for (uint32_t b = wq; b < nact; b += NWARP) {
                const uint4 *row = reinterpret_cast<const uint4 *>(cntbuf + (size_t)b * 256u) + 2u * lq;
                uint4 x = __ldcg(row), y = __ldcg(row + 1);
                uint32_t v[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
                const bool before = b < bid;
#pragma unroll
                for (int j = 0; j < 8; j++) { tacc[j] += v[j]; bacc[j] += before ? v[j] : 0u; }
            }
#pragma unroll
            for (int j = 0; j < 8; j++) { sh.wcnt[wq][8u * lq + j] = tacc[j]; sh.ent[wq * 256u + 8u * lq + j] = bacc[j]; }
            __syncthreads();
            uint32_t base = sh.fill[tid], tot = 0;
#pragma unroll
            for (int ww = 0; ww < NWARP; ww++) { tot += sh.wcnt[ww][tid]; base += sh.ent[ww * 256u + tid]; }
            sh.base[tid] = base;
            __syncthreads();
            if (tb0 < tb1) {
                uint32_t s_cur[ITEMS], d_cur[ITEMS], s_nxt[ITEMS], d_nxt[ITEMS];
                tile_load_s(g, tb0 * TILE, s_cur);
                tile_load_pred(g, tb0 * TILE, d_cur);
                for (uint32_t t = tb0; t < tb1; t++) {
                    if (t + 1 < tb1) {                                        // prefetch under the ranking
                        tile_load_s(g, (t + 1) * TILE, s_nxt);
                        tile_load_pred(g, (t + 1) * TILE, d_nxt);
                    }
                    tile_scatter<SPASS>(A, sh, g, t * TILE, s_cur, d_cur);
#pragma unroll
                    for (int r = 0; r < ITEMS; r++) { s_cur[r] = s_nxt[r]; d_cur[r] = d_nxt[r]; }
                }
            }
            __syncthreads();
            sh.fill[tid] += tot;
        }
        if (tid == 0) { sh.st_c = sh.ns_c; sh.st_phase = sh.ns_phase; sh.st_begin = sh.ns_begin; }
        grid.sync();
    }
    if (bid == 0 && tid == 0) {     // step statistics of this launch (diagnostics, tools/induce_steps.py)
        A.err[4 + (SPASS ? 3 : 0)] = bigcount; A.err[5 + (SPASS ? 3 : 0)] = smallcount; A.err[6 + (SPASS ? 3 : 0)] = bigtiles;
    }
}

}  // namespace b200sa
