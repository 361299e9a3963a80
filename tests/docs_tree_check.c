/*
 * tests/docs_tree_check.c -- serial construction of the generalized suffix tree of b200sa_docs_tree
 * for inputs too large for the Python definition.  TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's insertion loop (to_suffix_tree, suffix_tree/src/lib.rs:392-505; restated for one
 * text in tests/tree_oracle.c) over G and glcp, with every suffix cut at its document's end
 * (len = end of the document - G[i]), extended so that a suffix whose string equals a node's
 * (L == len) becomes a terminal of that node instead of a new leaf:
 *   climb from the node of the previous suffix to the deepest ancestor v with path_len(v) <= L;
 *   path_len(v) == L: L == len: v gains terminal i; else v gets a new leaf child of path length len;
 *   path_len(v) <  L: v's last child r is cut by a new node w of path length L that takes r;
 *                     L == len: w gains terminal i; else w also gets a new leaf child.
 * A new child is always the largest, so children stay in byte order in a doubly linked list.
 *
 * Document counts are computed independently of Hui's lowest-common-ancestor method: with prev[i] the
 * previous rank of the same document, the distinct documents of [lo, hi) are (hi - lo) minus the
 * number of i in [lo, hi) with prev[i] >= lo, counted offline with a Fenwick tree over the nodes in
 * reverse preorder (sa_lo does not increase).
 *
 * docs_tree_check fills the eight arrays of b200sa_docs_tree_out in preorder (cap >= 2n + 1 entries
 * each) and returns N, or -1 when the input is not a (G, glcp) pair the loop can take, -2 on an
 * allocation failure, -3 when the terminals met in preorder are not G in order.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NIL 0xFFFFFFFFu

typedef struct {
    uint32_t *parent, *plen, *tfirst, *tcount, *first, *last, *prev, *next;
    uint32_t count;
} tree_t;

static uint32_t new_node(tree_t *t, uint32_t plen)
{
    uint32_t v = t->count++;
    t->parent[v] = NIL; t->plen[v] = plen; t->tfirst[v] = NIL; t->tcount[v] = 0;
    t->first[v] = t->last[v] = t->prev[v] = t->next[v] = NIL;
    return v;
}

static void append_child(tree_t *t, uint32_t p, uint32_t c)
{
    t->parent[c] = p;
    t->prev[c] = t->last[p];
    t->next[c] = NIL;
    if (t->last[p] == NIL) t->first[p] = c; else t->next[t->last[p]] = c;
    t->last[p] = c;
}

static uint32_t pop_last_child(tree_t *t, uint32_t p)
{
    uint32_t c = t->last[p];
    if (c == NIL) return NIL;
    t->last[p] = t->prev[c];
    if (t->last[p] == NIL) t->first[p] = NIL; else t->next[t->last[p]] = NIL;
    t->prev[c] = NIL;
    return c;
}

static void add_terminal(tree_t *t, uint32_t v, uint32_t i)
{
    if (t->tcount[v]++ == 0) t->tfirst[v] = i;
}

static uint64_t doc_of(const uint32_t *starts, uint64_t ndocs, uint64_t p)
{
    uint64_t lo = 0, hi = ndocs;                  /* last d with starts[d] <= p */
    while (hi - lo > 1) {
        uint64_t mid = lo + (hi - lo) / 2;
        if (starts[mid] <= p) lo = mid; else hi = mid;
    }
    return lo;
}

int64_t docs_tree_check(uint64_t n64, const uint32_t *g, const uint32_t *glcp, const uint32_t *starts, uint64_t ndocs,
                        uint64_t cap, uint32_t *parent, uint32_t *depth, uint32_t *sa_lo, uint32_t *sa_hi,
                        uint32_t *label_start, uint32_t *subtree_end, uint32_t *term_end, uint32_t *doc_count)
{
    const uint32_t n = (uint32_t)n64;
    const uint32_t M = 2 * n + 1;
    if (cap < M || (n > 0 && ndocs == 0)) return -1;
    tree_t t;
    uint32_t **arrs[] = {&t.parent, &t.plen, &t.tfirst, &t.tcount, &t.first, &t.last, &t.prev, &t.next};
    const size_t na = sizeof arrs / sizeof arrs[0];
    int64_t rc = 0;
    for (size_t k = 0; k < na; k++) *arrs[k] = (uint32_t *)malloc((size_t)M * 4);
    uint32_t *order = (uint32_t *)malloc((size_t)M * 4), *id = (uint32_t *)malloc((size_t)M * 4);
    uint32_t *nxt = (uint32_t *)malloc(((size_t)n + 1) * 4), *fen = (uint32_t *)calloc((size_t)n + 1, 4);
    uint32_t *lastr = (uint32_t *)malloc((ndocs ? ndocs : 1) * 4);
    for (size_t k = 0; k < na; k++) if (!*arrs[k]) rc = -2;
    if (!order || !id || !nxt || !fen || !lastr) rc = -2;
    if (rc) goto out;
    t.count = 0;
    uint32_t root = new_node(&t, 0), last = root;
    for (uint32_t i = 0; i < n; i++) {
        uint32_t s = g[i], L = glcp[i];
        if (s >= n) { rc = -1; goto out; }
        uint64_t d = doc_of(starts, ndocs, s);
        uint32_t len = (uint32_t)((d + 1 < ndocs ? starts[d + 1] : n) - s);
        if (L > len || (i == 0 && L != 0) || L > t.plen[last]) { rc = -1; goto out; }
        uint32_t v = last;
        while (t.plen[v] > L && t.parent[v] != NIL) v = t.parent[v];
        if (t.plen[v] < L) {                      /* cut v's last child at depth L */
            uint32_t r = pop_last_child(&t, v);
            if (r == NIL) { rc = -1; goto out; }
            uint32_t w = new_node(&t, L);
            append_child(&t, w, r);
            append_child(&t, v, w);
            v = w;
        }
        if (L == len) {
            add_terminal(&t, v, i);
            last = v;
        } else {
            uint32_t leaf = new_node(&t, len);
            add_terminal(&t, leaf, i);
            append_child(&t, v, leaf);
            last = leaf;
        }
    }
    /* preorder: first child, else next sibling of the nearest ancestor that has one */
    uint32_t N = 0;
    for (uint32_t v = root; v != NIL;) {
        id[v] = N;
        order[N++] = v;
        if (t.first[v] != NIL) { v = t.first[v]; continue; }
        while (v != NIL && t.next[v] == NIL) v = t.parent[v];
        if (v != NIL) v = t.next[v];
    }
    uint32_t seen = 0;
    for (uint32_t k = 0; k < N; k++) {
        uint32_t v = order[k];
        if (t.tcount[v] && t.tfirst[v] != seen) { rc = -3; goto out; }
        sa_lo[k] = seen;
        term_end[k] = seen + t.tcount[v];
        seen += t.tcount[v];
        subtree_end[k] = 1;                       /* subtree size and terminals for now */
        sa_hi[k] = t.tcount[v];
    }
    for (uint32_t k = N; k-- > 1;) {
        uint32_t p = id[t.parent[order[k]]];
        subtree_end[p] += subtree_end[k];
        sa_hi[p] += sa_hi[k];
    }
    for (uint32_t k = 0; k < N; k++) {
        uint32_t v = order[k];
        subtree_end[k] += k;
        sa_hi[k] += sa_lo[k];
        parent[k] = k == 0 ? NIL : id[t.parent[v]];
        depth[k] = t.plen[v];
        label_start[k] = k == 0 ? 0 : g[sa_lo[k]] + t.plen[t.parent[v]];
    }
    /* doc counts: nxt[j] = next rank of the same document (NIL if none) */
    for (uint64_t d = 0; d < ndocs; d++) lastr[d] = NIL;
    for (uint32_t i = 0; i < n; i++) {
        uint64_t d = doc_of(starts, ndocs, g[i]);
        nxt[i] = NIL;
        if (lastr[d] != NIL) nxt[lastr[d]] = i;
        lastr[d] = i;
    }
    uint32_t cur = n;
    for (uint32_t k = N; k-- > 0;) {
        while (cur > sa_lo[k]) {                  /* ranks i whose prev is >= sa_lo[k] enter the tree */
            cur--;
            if (nxt[cur] != NIL)
                for (uint32_t x = nxt[cur] + 1; x <= n; x += x & (0u - x)) fen[x]++;
        }
        uint32_t c = 0;
        for (uint32_t x = sa_hi[k]; x > 0; x -= x & (0u - x)) c += fen[x];
        for (uint32_t x = sa_lo[k]; x > 0; x -= x & (0u - x)) c -= fen[x];
        doc_count[k] = (sa_hi[k] - sa_lo[k]) - c;
    }
    rc = N;
out:
    for (size_t k = 0; k < na; k++) free(*arrs[k]);
    free(order);
    free(id);
    free(nxt);
    free(fen);
    free(lastr);
    return rc;
}
