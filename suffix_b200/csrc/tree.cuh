// tree.cuh -- the suffix tree of the reference's suffix_tree crate, built from SA + LCP
// (SURVEY 8f-5; reference to_suffix_tree, suffix_tree/src/lib.rs:392-505).
//
// The reference inserts the suffixes in SA order into a pointer tree.  The same tree, node for node,
// follows from the LCP intervals (rules 1-8 of include/b200sa.h):
//   internal node  one per boundary i in [1, n) with lcp[i] > 0 that is the leftmost boundary of its
//                  interval (pse[i] == psv[i]); range [psv[i], nsv[i]), string depth lcp[i]
//   leaf           one per rank r that is not "merged" (suffix sa[r] is a proper prefix of sa[r+1]:
//                  lcp[r+1] == n - sa[r], the suffix then ends at the internal node of boundary r+1);
//                  range [r, r+1), string depth n - sa[r]
//   root           range [0, n), depth 0
// Preorder (the reference's, lexicographic) is the ascending order of the keys (sa_lo, depth).
#pragma once
#include "pipeline_kernels.cuh"

namespace b200sa {

constexpr uint32_t TREE_NONE = 0xffffffffu;
// bits of the check word (b200sa_suffix_tree_dev reports them through last_error)
constexpr uint32_t TREE_BAD_SA = 1, TREE_BAD_LCP0 = 2, TREE_BAD_LCP = 4, TREE_BAD_PARENT = 8, TREE_BAD_FIRST = 16;

// psv of every rank (exactly k_ansv's), and for the representative boundaries (rule 2) their nsv.
// rep[i] = 1 iff i is representative; the non-strict left search (pse) is only run where lcp[i] > 0.
__global__ void __launch_bounds__(BLK) k_tree_ansv(AnsvLevels L, uint64_t n, uint32_t *psv, uint32_t *nsv,
                                                   uint8_t *rep) {
    uint64_t i = (uint64_t)blockIdx.x * BLK + threadIdx.x;
    if (i >= n) return;
    uint32_t v = L.lv[0][i];
    uint32_t p = ansv_left<true>(L, i, v);
    psv[i] = p;
    bool r = i > 0 && v > 0 && p != ANSV_NONE && ansv_left<false>(L, i, v) == p;
    rep[i] = r ? 1 : 0;
    if (r) nsv[i] = (uint32_t)ansv_right(L, i, v, n);
}

__device__ __forceinline__ bool tree_merged(const uint32_t *sa, const uint32_t *lcp, uint32_t n, uint32_t r) {
    return r + 1 < n && lcp[r + 1] == n - sa[r];
}

// Scan input: nodes emitted by rank r (its representative internal node, its leaf), plus the input
// checks.  Every check runs before a value of sa or lcp is used to address memory (none is, before
// the host has read the check word back).
struct TreeCount {
    const uint32_t *sa, *lcp;
    const uint8_t *rep;
    uint32_t n;
    uint32_t *flag;
    __device__ uint32_t operator()(uint64_t i) const {
        uint32_t r = (uint32_t)i, s = sa[r], l = lcp[r], bad = 0;
        if (s >= n) bad |= TREE_BAD_SA;
        else if (l > n - s) bad |= TREE_BAD_LCP;
        if (r == 0 && l != 0) bad |= TREE_BAD_LCP0;
        if (r > 0) {
            uint32_t s1 = sa[r - 1];
            if (s1 < n && l > n - s1) bad |= TREE_BAD_LCP;
        }
        if (bad) atomicOr(flag, bad);
        return (uint32_t)rep[r] + (tree_merged(sa, lcp, n, r) ? 0u : 1u);
    }
};
// Scan output: key (sa_lo << B | depth) and payload sa_hi of each node; the root goes last.
struct TreeEmit {
    const uint32_t *sa, *lcp, *psv, *nsv;
    const uint8_t *rep;
    uint32_t n;
    int B;
    uint64_t *key;
    uint32_t *hi;
    __device__ void operator()(uint64_t i, uint32_t exc, uint32_t v) const {
        uint32_t r = (uint32_t)i, o = exc;
        uint32_t isrep = rep[r];
        if (isrep) {
            key[o] = ((uint64_t)psv[r] << B) | lcp[r];
            hi[o] = nsv[r];
            o++;
        }
        if (v > isrep) {
            key[o] = ((uint64_t)r << B) | (n - sa[r]);
            hi[o] = r + 1;
            o++;
        }
        if (r == n - 1) {
            key[o] = (uint64_t)0;
            hi[o] = n;
        }
    }
};

// first[l] = smallest preorder id whose sa_lo is l (the root's 0 for l = 0); first[n] = N.
__global__ void __launch_bounds__(BLK) k_tree_first(const uint64_t *key, uint32_t N, int B, uint32_t n,
                                                    uint32_t *first) {
    uint32_t j = blockIdx.x * BLK + threadIdx.x;
    if (j >= N) return;
    uint32_t l = (uint32_t)(key[j] >> B);
    if (j == 0 || (uint32_t)(key[j - 1] >> B) != l) first[l] = j;
    if (j == N - 1) first[n] = N;
}

struct TreeOut {
    uint32_t *parent, *depth, *sa_lo, *sa_hi, *label_start, *subtree_end;
};

// One thread per node: decode the key, find the parent (rule 5) by a binary search on depth among the
// nodes that start at plo, label start (rule 6) and subtree end (rule 7).  Threads v <= n also check
// that every rank starts some node.
__global__ void __launch_bounds__(BLK) k_tree_nodes(const uint64_t *key, const uint32_t *hiv, uint32_t N,
                                                    int B, const uint32_t *sa, const uint32_t *lcp,
                                                    const uint32_t *psv, const uint32_t *first, uint32_t n,
                                                    TreeOut o, uint32_t *flag) {
    uint32_t v = blockIdx.x * BLK + threadIdx.x;
    if (v <= n && first[v] == TREE_NONE) atomicOr(flag, TREE_BAD_FIRST);
    if (v >= N) return;
    const uint64_t mask = ((uint64_t)1 << B) - 1;
    uint64_t k = key[v];
    uint32_t lo = (uint32_t)(k >> B), d = (uint32_t)(k & mask), hi = hiv[v];
    uint32_t par = TREE_NONE, ls = 0, se = N;
    if (v > 0) {
        uint32_t llo = lcp[lo], lhi = hi < n ? lcp[hi] : 0u;
        uint32_t pd = llo > lhi ? llo : lhi;
        par = 0;
        if (pd > 0) {
            uint32_t plo = lhi > llo ? lo : psv[lo];
            uint32_t a = plo < n ? first[plo] : TREE_NONE, b = plo < n ? first[plo + 1] : TREE_NONE;
            uint64_t want = ((uint64_t)plo << B) | pd;
            bool found = false;
            if (a != TREE_NONE && b != TREE_NONE && a < b && b <= N) {
                while (a < b) {                       // lower bound of want in key[a, b)
                    uint32_t m = a + (b - a) / 2;
                    if (key[m] < want) a = m + 1; else b = m;
                }
                found = a < N && key[a] == want;
            }
            if (found) par = a;
            else atomicOr(flag, TREE_BAD_PARENT);
        }
        ls = sa[lo] + pd;
        if (hi < n) {
            se = first[hi];
            if (se == TREE_NONE) se = N;              // flagged above by thread hi
        }
    }
    o.parent[v] = par;
    o.depth[v] = d;
    o.sa_lo[v] = lo;
    o.sa_hi[v] = hi;
    o.label_start[v] = ls;
    o.subtree_end[v] = se;
}

}  // namespace b200sa
