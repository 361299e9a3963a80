/*
 * tests/tree_oracle.c -- CPU restatement of the reference's suffix tree construction
 * (to_suffix_tree, suffix_tree/src/lib.rs:392-505).  TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The suffixes are inserted in SA order.  For suffix i with lcp[i] = L, climb from the last
 * inserted leaf to the deepest ancestor v with path_len(v) <= L (the root if none).
 *   path_len(v) == L: v gets a new leaf child, label [sa[i] + L, n), terminal sa[i].
 *   path_len(v) <  L: v's last child r is cut; a new internal node w with path length L and label
 *                     [sa[i-1] + path_len(v), sa[i-1] + L) takes r (whose label is rewritten to
 *                     [sa[i-1] + L, sa[i-1] + path_len(r))) and the new leaf, and replaces r as
 *                     v's last child.
 * Children are kept in byte order because a new child is always the largest and a split pops the
 * last one, so each node needs only a doubly linked child list.  Everything is iterative: a^n is
 * n levels deep.
 *
 * oracle_suffix_tree flattens the tree to the arrays of b200sa_tree in preorder (children in byte
 * order) plus the oracle's own label offsets and terminals:
 *   parent, depth (path_len), sa_lo, sa_hi, label_start (= sa[sa_lo] + depth of the parent,
 *   the canonical offset), subtree_end, own_start, own_end, terminal (0xFFFFFFFF: none; the
 *   root's is n).  Every array holds cap >= 2n + 1 entries.  Returns N, or -1 when the input is
 *   not an SA/LCP pair the loop can take, -2 on allocation failure.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NIL 0xFFFFFFFFu

typedef struct {
    uint32_t *parent, *start, *end, *plen, *term, *first, *last, *prev, *next;
    uint32_t count;
} tree_t;

static uint32_t new_node(tree_t *t, uint32_t start, uint32_t end, uint32_t term)
{
    uint32_t v = t->count++;
    t->parent[v] = NIL; t->start[v] = start; t->end[v] = end; t->plen[v] = 0; t->term[v] = term;
    t->first[v] = t->last[v] = t->prev[v] = t->next[v] = NIL;
    return v;
}

static void set_parent(tree_t *t, uint32_t v, uint32_t p)
{
    t->parent[v] = p;
    t->plen[v] = t->plen[p] + (t->end[v] - t->start[v]);
}

static void append_child(tree_t *t, uint32_t p, uint32_t c)
{
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

int64_t oracle_suffix_tree(uint64_t n64, const uint32_t *sa, const uint32_t *lcp, uint64_t cap,
                           uint32_t *parent, uint32_t *depth, uint32_t *sa_lo, uint32_t *sa_hi,
                           uint32_t *label_start, uint32_t *subtree_end,
                           uint32_t *own_start, uint32_t *own_end, uint32_t *terminal)
{
    const uint32_t n = (uint32_t)n64;
    const uint32_t M = 2 * n + 1;
    if (cap < M) return -1;
    tree_t t;
    uint32_t **arrs[] = {&t.parent, &t.start, &t.end, &t.plen, &t.term, &t.first, &t.last, &t.prev, &t.next};
    int64_t rc = 0;
    for (size_t k = 0; k < sizeof arrs / sizeof arrs[0]; k++) *arrs[k] = (uint32_t *)malloc((size_t)M * 4);
    uint32_t *order = (uint32_t *)malloc((size_t)M * 4), *id = (uint32_t *)malloc((size_t)M * 4);
    for (size_t k = 0; k < sizeof arrs / sizeof arrs[0]; k++) if (!*arrs[k]) rc = -2;
    if (!order || !id) rc = -2;
    if (rc) goto out;
    t.count = 0;
    uint32_t root = new_node(&t, 0, 0, n), last = root;
    for (uint32_t i = 0; i < n; i++) {
        uint32_t s = sa[i], L = lcp[i];
        if (s >= n || L > n - s || (i == 0 && L != 0)) { rc = -1; goto out; }
        uint32_t v = last;
        while (t.plen[v] > L && t.parent[v] != NIL) v = t.parent[v];
        uint32_t dv = t.plen[v];
        uint32_t leaf = new_node(&t, s + L, n, s);
        if (dv == L) {
            set_parent(&t, leaf, v);
            append_child(&t, v, leaf);
        } else {                                  /* dv < L */
            uint32_t r = pop_last_child(&t, v), p = sa[i - 1];
            if (r == NIL || L > n - p) { rc = -1; goto out; }
            uint32_t w = new_node(&t, p + dv, p + L, NIL);
            set_parent(&t, w, v);
            t.start[r] = p + L;
            t.end[r] = p + t.plen[r];
            set_parent(&t, r, w);
            set_parent(&t, leaf, w);
            append_child(&t, w, r);
            append_child(&t, w, leaf);
            append_child(&t, v, w);
        }
        last = leaf;
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
    /* sa_lo: terminals (the root's aside) met before the node in preorder; sizes bottom-up */
    uint32_t seen = 0;
    for (uint32_t k = 0; k < N; k++) {
        uint32_t v = order[k];
        sa_lo[k] = seen;
        if (k > 0 && t.term[v] != NIL) seen++;
        subtree_end[k] = 1;                       /* subtree size for now */
        sa_hi[k] = (k > 0 && t.term[v] != NIL) ? 1 : 0;
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
        own_start[k] = t.start[v];
        own_end[k] = t.end[v];
        terminal[k] = t.term[v];
        label_start[k] = k == 0 ? 0 : sa[sa_lo[k]] + t.plen[t.parent[v]];
    }
    rc = N;
out:
    for (size_t k = 0; k < sizeof arrs / sizeof arrs[0]; k++) free(*arrs[k]);
    free(order);
    free(id);
    return rc;
}

/* First node k in [1, N) whose label text[a[k], a[k] + len[k]) differs from text[b[k], ...), or -1.
 * Equal offsets name equal bytes; leaves (whose labels run to the end of the text, O(n^2) bytes in
 * all) always have equal offsets, so only internal nodes are compared byte by byte. */
int64_t oracle_tree_labels_differ(const uint8_t *text, uint64_t N, const uint32_t *a, const uint32_t *b,
                                  const uint32_t *len)
{
    for (uint64_t k = 1; k < N; k++)
        if (a[k] != b[k] && memcmp(text + a[k], text + b[k], len[k]) != 0) return (int64_t)k;
    return -1;
}
