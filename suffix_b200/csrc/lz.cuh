// lz.cuh -- the longest previous factor of every position and the LZ77 factorization it defines
// (DESIGN 6b f-12), from the table R (sa or G) and its LCP array lam alone.
//
// LPF (Crochemore & Ilie 2008): for the rank r with R[r] = p, psv(r) / nsv(r) are the nearest ranks on
// either side whose position is below p, found by ansv_left / ansv_right over the block minima of R.
// The longest prefix S_p shares with an earlier suffix is the longer of its LCPs with those two, each the
// range minimum of lam between the ranks (docs_range_min over the block minima of lam).  glcp never
// crosses a document end, so the same kernel serves documents.
//
// Parse (Shun & Zhao 2013): next(p) = p + max(1, lpf[p]) is a forest on [0, n] rooted at n; the factor
// starts are the path of 0.  J starts as next and is squared every round (J <- J o J, into the other
// buffer); before squaring, every marked p with J[p] < n marks J[p].  After round k the marks hold the
// first 2^k factor starts, so the round that finds J[0] >= n -- ceil(log2 z) rounds in -- ends the parse.
// Marks are set in place: a mark read early or late is still a start on 0's path.  The host launches
// the bound bit_length(n) rounds without syncing; the round that sees J[0] >= n raises a flag that
// makes every later launch return at once.
#pragma once
#include "docs.cuh"

namespace b200sa {

constexpr uint32_t LZ_LITERAL = 0xffffffffu;

// one thread per rank; lpf[p] and (src non-null) src[p] at p = R[r]
__global__ void __launch_bounds__(BLK) k_lz_lpf(AnsvLevels LR, AnsvLevels LL, uint32_t n, uint32_t *lpf,
                                                uint32_t *src) {
    const uint64_t r = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (r >= n) return;
    const uint32_t p = LR.lv[0][r];
    const uint32_t a = ansv_left<true>(LR, r, p);
    const uint64_t b = ansv_right(LR, r, p, n);
    const uint32_t lL = a != ANSV_NONE ? docs_range_min(LL, (uint64_t)a + 1, r, 0xffffffffu) : 0u;
    const uint32_t lR = b < n ? docs_range_min(LL, r + 1, b, 0xffffffffu) : 0u;
    lpf[p] = lL > lR ? lL : lR;
    if (src) src[p] = (lL >= lR && lL > 0) ? LR.lv[0][a] : (lR > 0 ? LR.lv[0][b] : LZ_LITERAL);
}

// J[p] = next(p) for p < n, J[n] = n; mark 0 (the bitmap is zeroed before)
__global__ void __launch_bounds__(BLK) k_lz_next(const uint32_t *__restrict__ lpf, uint32_t n, uint32_t *J,
                                                 uint32_t *marks) {
    const uint64_t p = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (p > n) return;
    if (p == n) {
        J[p] = n;
        return;
    }
    const uint32_t l = lpf[p];
    J[p] = (uint32_t)p + (l > 1 ? l : 1u);
    if (p == 0) marks[0] = 1u;
}

// state[0]: the parse is done; state[1]: rounds squared so far.  One thread per bitmap word.
__global__ void __launch_bounds__(BLK) k_lz_mark(const uint32_t *__restrict__ J, uint32_t n, uint32_t *marks,
                                                 uint32_t nwords, uint32_t *state) {
    const uint32_t w = blockIdx.x * BLK + threadIdx.x;
    if (state[0] || J[0] >= n) {            // every start is marked: J[0] = f_(2^k) >= n after round k
        if (w == 0) state[0] = 1u;
        return;
    }
    if (w >= nwords) return;
    for (uint32_t m = marks[w]; m; m &= m - 1) {
        const uint32_t q = J[w * 32u + (uint32_t)(__ffs(m) - 1)];
        if (q < n) atomicOr(marks + (q >> 5), 1u << (q & 31));
    }
}

// Jn = J o J over [0, n]
__global__ void __launch_bounds__(BLK) k_lz_square(const uint32_t *__restrict__ J, uint32_t n, uint32_t *Jn,
                                                   uint32_t *state) {
    const uint64_t p = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (p > n || state[0]) return;
    Jn[p] = J[J[p]];
    if (p == 0) state[1]++;
}

// ---- count and emit, one scan element per bitmap word (InPopcWords counts)
struct LzNoOut {
    __device__ void operator()(uint64_t, uint32_t, uint32_t) const {}
};
struct LzEmitOut {
    const uint32_t *marks, *lpf, *src;
    uint32_t *start, *len, *fsrc;
    __device__ void operator()(uint64_t w, uint32_t exc, uint32_t v) const {
        if (!v) return;
        uint32_t k = exc;
        for (uint32_t m = marks[w]; m; m &= m - 1, k++) {
            const uint32_t p = (uint32_t)w * 32u + (uint32_t)(__ffs(m) - 1), l = lpf[p];
            start[k] = p;
            len[k] = l > 1 ? l : 1u;
            fsrc[k] = src[p];
        }
    }
};

}  // namespace b200sa
