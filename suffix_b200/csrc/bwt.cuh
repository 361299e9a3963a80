// bwt.cuh -- the Burrows-Wheeler transform of a text or of many documents and its inverse (DESIGN 6b f-13).
//
// Rows: the k terminator rows $_d D_d first, then row k + r for the rotation at G[r] (sa for one text).
// Forward: one thread per row gathers its L symbol (a byte, or the terminator $_d as 256 + d), the
// terminator rows are compacted out by a look-back scan over their flag bitmap, and r counts the rows
// whose symbol differs from the one before.
//
// Inverse: psi = LF^-1.  psi(d) = term_rows[d] for d < k; the non-terminator rows of L, stably sorted by
// byte (one 8-bit sort_pairs pass over (byte, index u in bwt)), give psi(k + j) = row(u_j) and F[k + j].
// row(u) = u + #{i : t_(i) - i <= u} over the sorted term rows t.  psi(x) and the byte of row psi(x) are
// interleaved in one u64 per row, so one walk step is one dependent load.
// List ranking with rulers: the rows below k and the rows whose hash falls below 2^32 / s are rulers.
// Each ruler walks psi to the next ruler (its segment); pointer doubling over the ruler list, broken at
// the rulers below k, gives every ruler the document it belongs to and the bytes left to its document's
// end; each ruler then walks its segment again and writes its bytes.  The input is valid iff every
// terminator ruler's list ends at itself and the segments of the rulers whose list ends at a terminator
// cover all n + k rows.
#pragma once
#include "docs.cuh"

namespace b200sa {

constexpr uint32_t BWT_TERM_F = 0x100u;          // F of a terminator row in the interleaved psi / F array

// ---- forward
// The row layout over (starts, k): starts == null is one text (k = 1, starts = [0]).
struct BwtRows {
    const uint8_t *text;
    const uint32_t *sa, *starts;
    uint32_t n, k;
    __device__ __forceinline__ uint32_t start(uint32_t d) const { return starts ? __ldg(starts + d) : 0u; }
    __device__ __forceinline__ uint32_t end(uint32_t d) const { return d + 1 < k ? start(d + 1) : n; }
    // L of row i: a byte, or 256 + d for $_d
    __device__ __forceinline__ uint32_t sym(uint32_t i) const {
        if (i < k) {
            const uint32_t e = end(i);
            return e > start(i) ? (uint32_t)__ldg(text + e - 1) : 256u + i;
        }
        const uint32_t p = __ldg(sa + (i - k));
        const uint32_t d = starts ? docs_find(starts, k, p) : 0u;
        return p == start(d) ? 256u + d : (uint32_t)__ldg(text + p - 1);
    }
};

// One thread per row: lbyte[i] = L's byte (any value on a terminator row), the terminator bitmap, the
// term row of each document, and (runs non-null) the number of rows whose symbol differs from the one
// before, row 0 counting as a run start.
__global__ void __launch_bounds__(BLK) k_bwt_gather(BwtRows R, uint32_t nrows, uint8_t *lbyte, uint32_t *term_bm,
                                                    uint32_t *term_rows, unsigned long long *runs) {
    __shared__ uint32_t s_runs[NWARP];
    const uint32_t i = blockIdx.x * BLK + threadIdx.x, l = lane_id();
    const bool in = i < nrows;
    const uint32_t s = in ? R.sym(i) : 0u;
    const bool term = in && s >= 256u;
    if (in) {
        lbyte[i] = (uint8_t)s;
        if (term) term_rows[s - 256u] = i;
    }
    const uint32_t bits = __ballot_sync(FULL, term);
    if (l == 0 && i < nrows) term_bm[i >> 5] = bits;
    if (!runs) return;
    uint32_t prev = __shfl_up_sync(FULL, s, 1);
    if (l == 0 && in && i > 0) prev = R.sym(i - 1);
    const uint32_t head = __popc(__ballot_sync(FULL, in && (i == 0 || s != prev)));
    if (l == 0) s_runs[warp_id()] = head;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < NWARP; w++) t += s_runs[w];
        if (t) atomicAdd(runs, (unsigned long long)t);
    }
}

// Scan output over terminator-bitmap words (InPopcWords counts the terminators): the bytes of word w's
// non-terminator rows go to bwt[row - terminators before row].
struct BwtCompactOut {
    const uint32_t *term_bm;
    const uint8_t *lbyte;
    uint8_t *bwt;
    uint32_t nrows;
    __device__ void operator()(uint64_t w, uint32_t exc, uint32_t) const {
        const uint32_t bm = term_bm[w], row0 = (uint32_t)w * 32u;
        uint32_t u = row0 - exc;
        for (uint32_t b = 0; b < 32u && row0 + b < nrows; b++)
            if (!((bm >> b) & 1u)) bwt[u++] = lbyte[row0 + b];
    }
};

// ---- inverse
// Sort key of index u of the bwt: its byte.
struct BwtByteKey {
    const uint8_t *bwt;
    __device__ __forceinline__ uint32_t operator()(uint64_t u) const { return bwt[u]; }
};

// Sorted term rows ts[0, k): words[0] |= 1 if one is >= nrows or two are equal.
__global__ void __launch_bounds__(BLK) k_bwt_terms_check(const uint32_t *__restrict__ ts, uint32_t k, uint32_t nrows,
                                                         uint32_t *words) {
    const uint32_t i = blockIdx.x * BLK + threadIdx.x;
    const bool bad = i < k && (ts[i] >= nrows || (i > 0 && ts[i - 1] == ts[i]));
    if (__any_sync(FULL, bad) && lane_id() == 0) atomicOr(words, 1u);
}

// pf[x] = F(psi(x)) << 32 | psi(x) for every row x < nrows = n + k: a walk step reads the next row and
// its byte in one load.  fk / fu: the bwt bytes stably sorted and their indices u; F(y) = fk[y - k], or
// BWT_TERM_F for y < k.  ts: the sorted term rows.
__global__ void __launch_bounds__(BLK) k_bwt_psi(const uint32_t *__restrict__ term_rows, const uint32_t *__restrict__ ts,
                                                 uint32_t k, const uint32_t *__restrict__ fk,
                                                 const uint32_t *__restrict__ fu, uint32_t nrows,
                                                 unsigned long long *pf) {
    const uint32_t x = blockIdx.x * BLK + threadIdx.x;
    if (x >= nrows) return;
    uint32_t y;
    if (x < k) {
        y = term_rows[x];
    } else {
        const uint32_t u = fu[x - k];
        uint32_t lo = 0, hi = k;                       // #{i : ts[i] - i <= u}; ts[i] - i never decreases
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (__ldg(ts + mid) - mid <= u) lo = mid + 1; else hi = mid;
        }
        y = u + lo;
    }
    pf[x] = ((unsigned long long)(y < k ? BWT_TERM_F : fk[y - k]) << 32) | y;
}

// Rulers: the rows below k, and the rows whose hash is below 2^32 / s when s <= n (a spacing above n
// leaves the terminator rows alone).
struct BwtRuler {
    uint32_t k, s;
    bool hashed;
    __device__ __forceinline__ static uint32_t mix(uint32_t x) {
        x ^= x >> 16;
        x *= 0x7feb352du;
        x ^= x >> 15;
        x *= 0x846ca68bu;
        x ^= x >> 16;
        return x;
    }
    __device__ __forceinline__ bool operator()(uint32_t row) const {
        return row < k || (hashed && __umulhi(mix(row), s) == 0u);
    }
};

__global__ void __launch_bounds__(BLK) k_bwt_ruler_bits(BwtRuler isr, uint32_t nrows, uint32_t *bm) {
    const uint32_t x = blockIdx.x * BLK + threadIdx.x;
    const uint32_t bits = __ballot_sync(FULL, x < nrows && isr(x));
    if (lane_id() == 0 && x < nrows) bm[x >> 5] = bits;
}

// One thread per ruler-bitmap word w: the ruler rows in order, rrow[wpre[w] + i] for its i-th set bit
// (wpre: the exclusive prefix of the words' popcounts).
__global__ void __launch_bounds__(BLK) k_bwt_ruler_list(const uint32_t *__restrict__ bm, const uint32_t *__restrict__ wpre,
                                                        uint32_t nwords, uint32_t *rrow) {
    const uint32_t w = blockIdx.x * BLK + threadIdx.x;
    if (w >= nwords) return;
    uint32_t j = wpre[w];
    for (uint32_t m = bm[w]; m; m &= m - 1) rrow[j++] = w * 32u + (uint32_t)(__ffs(m) - 1);
}

// One thread per ruler j: walk psi to the next ruler e.  nv[j] = val << 32 | nxt: a terminator e ends the
// list (nxt = e < k, val = steps - 1 bytes); otherwise nxt = e's ruler index (>= k) and val = steps bytes.
// steps[j] and the longest walk (words[1]) are kept for the validity check and the record.
__global__ void __launch_bounds__(BLK) k_bwt_walk(const unsigned long long *__restrict__ pf, BwtRuler isr,
                                                  const uint32_t *__restrict__ rrow, const uint32_t *__restrict__ bm,
                                                  const uint32_t *__restrict__ wpre, uint32_t m,
                                                  unsigned long long *nv, uint32_t *steps, uint32_t *words) {
    const uint32_t j = blockIdx.x * BLK + threadIdx.x;
    uint32_t st = 0;
    if (j < m) {
        uint32_t cur = rrow[j];
        do {
            cur = (uint32_t)pf[cur];
            st++;
        } while (!isr(cur));
        uint32_t nxt, val;
        if (cur < isr.k) {
            nxt = cur;
            val = st - 1;
        } else {
            nxt = wpre[cur >> 5] + __popc(bm[cur >> 5] & ((1u << (cur & 31)) - 1u));
            val = st;
        }
        nv[j] = ((unsigned long long)val << 32) | nxt;
        steps[j] = st;
    }
    st = __reduce_max_sync(FULL, st);
    if (lane_id() == 0 && st) atomicMax(words + 1, st);
}

// One round of pointer doubling, nv -> nv2: a ruler whose list has not ended takes its successor's val and
// nxt.  Round r runs only if round r - 1 moved a ruler (flags[r - 1]); a round that does not run copies.
__global__ void __launch_bounds__(BLK) k_bwt_jump(const unsigned long long *__restrict__ nv, uint32_t m, uint32_t k,
                                                  unsigned long long *nv2, uint32_t *flags, uint32_t r) {
    const uint32_t j = blockIdx.x * BLK + threadIdx.x;
    if (j >= m) return;
    unsigned long long v = nv[j];
    const uint32_t nxt = (uint32_t)v;
    const bool run = r == 0 || flags[r - 1] != 0u;
    const bool move = run && nxt >= k;
    if (move) {
        const unsigned long long q = nv[nxt];
        v = (((v >> 32) + (q >> 32)) << 32) | (uint32_t)q;
    }
    nv2[j] = v;
    if (move) flags[r] = 1u;
}

// Validity: *sum += the steps of the rulers whose list ends at a terminator; words[0] |= 2 if a terminator
// ruler's list ends at another one.
__global__ void __launch_bounds__(BLK) k_bwt_valid(const unsigned long long *__restrict__ nv,
                                                   const uint32_t *__restrict__ steps, uint32_t m, uint32_t k,
                                                   unsigned long long *sum, uint32_t *words) {
    const uint32_t j = blockIdx.x * BLK + threadIdx.x;
    uint32_t st = 0;
    bool bad = false;
    if (j < m) {
        const uint32_t nxt = (uint32_t)nv[j];
        if (nxt < k) st = steps[j];
        bad = j < k && nxt != j;
    }
    const uint32_t t = __reduce_add_sync(FULL, st);
    const bool anybad = __any_sync(FULL, bad);
    if (lane_id() == 0) {
        if (t) atomicAdd(sum, (unsigned long long)t);
        if (anybad) atomicOr(words, 2u);
    }
}

// Scan over the documents: starts[d] = exclusive sum of the document lengths (val of ruler d).
struct BwtLenIn {
    const unsigned long long *nv;
    __device__ uint32_t operator()(uint64_t d) const { return (uint32_t)(nv[d] >> 32); }
};
struct BwtStartsOut {
    uint32_t *starts, *starts_out;
    __device__ void operator()(uint64_t d, uint32_t exc, uint32_t) const {
        starts[d] = exc;
        if (starts_out) starts_out[d] = exc;
    }
};

// One thread per ruler: walk the segment again and write its bytes from the offset the ranking gave.
__global__ void __launch_bounds__(BLK) k_bwt_emit(const unsigned long long *__restrict__ pf,
                                                  const uint32_t *__restrict__ rrow, const uint32_t *__restrict__ steps,
                                                  const unsigned long long *__restrict__ nv,
                                                  const uint32_t *__restrict__ starts, uint32_t m, uint32_t k,
                                                  uint8_t *out) {
    const uint32_t j = blockIdx.x * BLK + threadIdx.x;
    if (j >= m) return;
    const unsigned long long v = nv[j];
    const uint32_t d = (uint32_t)v;
    uint32_t pos = starts[d] + (uint32_t)(nv[d] >> 32) - (uint32_t)(v >> 32);
    uint32_t cur = rrow[j];
    for (uint32_t s = steps[j]; s; s--) {
        const unsigned long long e = pf[cur];
        cur = (uint32_t)e;
        if (cur >= k) out[pos++] = (uint8_t)(e >> 32);
    }
}

}  // namespace b200sa
