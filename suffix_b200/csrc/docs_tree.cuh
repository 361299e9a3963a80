// docs_tree.cuh -- the generalized suffix tree of many documents (SURVEY 8f-7) and the number of
// distinct documents below every node, from G and glcp of b200sa_docs_build (docs.cuh).
//
// The tree is the one of tree.cuh with len[r] = document end - G[r] (DocsLen) and rule 3': a rank
// is also merged when its string equals the previous rank's.  On top of it:
//   term_end   the terminals of node v are G[sa_lo[v], term_end[v]): the last rank r of each run of
//              equal strings writes r + 1 at the node (a, len[r]), a = the first rank sharing len[r]
//              bytes with r (r itself, or ansv_left with threshold len[r]); other nodes keep sa_lo
//   doc_count  Hui's method: the ranks sorted stably by document give each rank its predecessor of
//              the same document; the pair (prev, i) adds 1 at their lowest common ancestor, the node
//              (lo, D) with D = min glcp(prev, i] and lo = ansv_left(prev + 1, D) (the root if D = 0);
//              doc_count[v] = ranks below v - pairs whose ancestor lies in v's subtree (a scan over ids)
#pragma once
#include "docs.cuh"
#include "tree.cuh"

namespace b200sa {

// Per rank: document and suffix length of G[r] (one search over doc_starts, reused by every stage).
// An out-of-range entry gets length 0; the tree's input check flags it.
__global__ void __launch_bounds__(BLK) k_dtree_len(const uint32_t *__restrict__ g, uint32_t n,
                                                   const uint32_t *__restrict__ starts, uint32_t ndocs,
                                                   uint32_t *len, uint32_t *doc) {
    uint32_t r = blockIdx.x * BLK + threadIdx.x;
    if (r >= n) return;
    uint32_t p = g[r], d = 0, l = 0;
    if (p < n) {
        d = docs_find(starts, ndocs, p);
        l = docs_end(starts, ndocs, n, d) - p;
    }
    len[r] = l;
    doc[r] = d;
}

// The last rank of each run of equal strings closes the terminals of its node.
__global__ void __launch_bounds__(BLK) k_dtree_term(AnsvLevels L, const uint32_t *__restrict__ len, uint32_t n,
                                                    const uint64_t *key, const uint32_t *first, uint32_t N, int B,
                                                    uint32_t *term_end, uint32_t *flag) {
    uint32_t r = blockIdx.x * BLK + threadIdx.x;
    if (r >= n) return;
    const uint32_t *glcp = L.lv[0];
    uint32_t lr = len[r];
    if (r + 1 < n && glcp[r + 1] == lr && len[r + 1] == lr) return;
    uint32_t a = glcp[r] < lr ? r : ansv_left<true>(L, r, lr);
    uint32_t v;
    if (a != ANSV_NONE && tree_find(key, first, N, B, n, a, lr, &v)) term_end[v] = r + 1;
    else atomicOr(flag, TREE_BAD_NODE);
}

// Index of a sorted item (the ranks are fed to the document sort in rank order).
struct LoadIndex {
    __device__ __forceinline__ uint32_t operator()(uint64_t i) const { return (uint32_t)i; }
};

// Item k of the ranks sorted by document (dk = documents, rk = ranks): the pair (rk[k-1], rk[k]) of
// one document adds 1 at its lowest common ancestor.  On repetitive text most pairs meet at the same
// few nodes, so equal targets are added once per warp, and the root's share once per block.
__global__ void __launch_bounds__(BLK) k_dtree_pairs(AnsvLevels L, const uint32_t *__restrict__ dk,
                                                     const uint32_t *__restrict__ rk, const uint32_t *__restrict__ len,
                                                     uint32_t n, const uint64_t *key, const uint32_t *first,
                                                     uint32_t N, int B, uint32_t *pairs_at, uint32_t *flag) {
    __shared__ uint32_t root_pairs;
    if (threadIdx.x == 0) root_pairs = 0;
    __syncthreads();
    uint32_t k = blockIdx.x * BLK + threadIdx.x, v = TREE_NONE;
    if (k > 0 && k < n && dk[k - 1] == dk[k]) {
        uint32_t p = rk[k - 1], i = rk[k];
        uint32_t D = docs_range_min(L, (uint64_t)p + 1, i, len[i]);
        if (D == 0) {
            v = 0;
        } else {
            uint32_t lo = ansv_left<true>(L, (uint64_t)p + 1, D);
            if (lo == ANSV_NONE || !tree_find(key, first, N, B, n, lo, D, &v)) atomicOr(flag, TREE_BAD_NODE);
        }
    }
    uint32_t at_root = __ballot_sync(FULL, v == 0);
    if (lane_id() == 0 && at_root) atomicAdd(&root_pairs, (uint32_t)__popc(at_root));
    uint32_t peers = __match_any_sync(FULL, v);
    if (v != 0 && v != TREE_NONE && lane_id() == (uint32_t)(__ffs(peers) - 1))
        atomicAdd(pairs_at + v, (uint32_t)__popc(peers));
    __syncthreads();
    if (threadIdx.x == 0 && root_pairs) atomicAdd(pairs_at, root_pairs);
}

// doc_count[v] = (sa_hi - sa_lo) - pairs inside v's subtree; P = exclusive scan of pairs_at over ids.
__global__ void __launch_bounds__(BLK) k_dtree_count(const uint32_t *__restrict__ sa_lo,
                                                     const uint32_t *__restrict__ sa_hi,
                                                     const uint32_t *__restrict__ subtree_end,
                                                     const uint32_t *__restrict__ P, uint32_t N, uint32_t *doc_count) {
    uint32_t v = blockIdx.x * BLK + threadIdx.x;
    if (v >= N) return;
    doc_count[v] = (sa_hi[v] - sa_lo[v]) - (P[subtree_end[v]] - P[v]);
}

// Document frequency of the ranges [start, end) of k_positions<DocsEnd>: 0 for an empty range, else
// doc_count of a node with that range.  The nodes that start at `start` are consecutive in preorder
// with sa_hi non-increasing (strictly below the root), so one binary search over [first id with
// sa_lo >= start, N) finds the first with sa_lo != start or sa_hi <= end.  A range no node has sets *flag.
__global__ void __launch_bounds__(BLK) k_dtree_counts(const uint32_t *__restrict__ sa_lo,
                                                      const uint32_t *__restrict__ sa_hi,
                                                      const uint32_t *__restrict__ cnt, uint32_t N,
                                                      const uint32_t *__restrict__ qs, const uint32_t *__restrict__ qe,
                                                      uint32_t nq, uint32_t *out, uint32_t *flag) {
    uint32_t q = blockIdx.x * BLK + threadIdx.x;
    if (q >= nq) return;
    uint32_t s = qs[q], e = qe[q], res = 0;
    if (s < e) {
        uint32_t a = 0, b = N;
        while (a < b) {                                   // first id with sa_lo >= s
            uint32_t m = a + (b - a) / 2;
            if (sa_lo[m] < s) a = m + 1; else b = m;
        }
        b = N;
        while (a < b) {                                   // first id in the chain with sa_hi <= e, or past it
            uint32_t m = a + (b - a) / 2;
            if (sa_lo[m] == s && sa_hi[m] > e) a = m + 1; else b = m;
        }
        if (a < N && sa_lo[a] == s && sa_hi[a] == e) res = cnt[a];
        else atomicOr(flag, 1u);
    }
    out[q] = res;
}

}  // namespace b200sa
