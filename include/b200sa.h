/*
 * b200sa.h -- C-ABI of the H100-native suffix-array / LCP construction engine.
 *
 * Drop-in boundary for the construction hot path of BurntSushi/suffix
 * (reference: src/table.rs of BurntSushi/suffix).  The reference has no FFI of its
 * own; the seam is the two private calls made by its public API:
 *
 *   SuffixTable::new      -> sais_table(&text)            src/table.rs:83, :378-386
 *   SuffixTable::lcp_lens -> lcp_lens_quadratic(text,sa)  src/table.rs:135, :348-361
 *
 * Every entry point takes plain pointers and sizes (no torch / C++ types).
 * Caller owns every buffer passed in; the library never retains host
 * pointers after return.  Device workspace is owned by the context and is
 * reused across calls.  A context is NOT thread-safe; distinct contexts are.
 * There is NO CPU fallback: without a usable CUDA device every call returns
 * B200SA_ERR_NO_DEVICE / B200SA_ERR_CUDA.
 *
 * Suffix indices are byte offsets stored as u32 (reference: src/table.rs:64-66).
 * The reference accepts n <= 2^32-1 (src/table.rs:380); this library accepts
 * n <= B200SA_MAX_N = 2^32-4096 (grid index arithmetic is done in u32 with
 * tile-sized slack) and returns B200SA_ERR_TOO_LARGE above that.
 */
#ifndef B200SA_H
#define B200SA_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200sa_ctx b200sa_ctx;

#define B200SA_MAX_N 0xFFFFF000ull

enum {
    B200SA_OK            =  0,
    B200SA_ERR_BAD_ARG   = -1,  /* null pointer / bad size / (lcp) table not a permutation of 0..n-1 */
    B200SA_ERR_TOO_LARGE = -2,  /* n > B200SA_MAX_N (reference panics above 2^32-1, src/table.rs:380) */
    B200SA_ERR_NO_DEVICE = -3,
    B200SA_ERR_OOM       = -4,
    B200SA_ERR_CUDA      = -5,
    B200SA_ERR_INTERNAL  = -6,  /* device-side invariant violated                 */
    B200SA_ERR_COMM      = -7   /* NCCL missing or a collective failed            */
};

/* Context: binds a CUDA device, one stream, the device workspace. */
int  b200sa_ctx_create(int device, b200sa_ctx **out);
void b200sa_ctx_destroy(b200sa_ctx *ctx);

/* ---- host-buffer entry points (what a Rust/C++ SuffixTable binds) ---- */

/* Replaces `sais_table(text) -> Vec<u32>` (src/table.rs:378-386), the body of
 * SuffixTable::new (src/table.rs:78-85).  text: n bytes (any bytes; UTF-8 is
 * handled at byte level exactly like the reference's `Utf8` wrapper,
 * src/table.rs:778-800).  sa_out: n u32, caller-allocated.  n==0 and n==1
 * succeed without launching (src/table.rs:395-402). */
int b200sa_build(b200sa_ctx *ctx, const uint8_t *text, uint64_t n, uint32_t *sa_out);

/* Replaces `lcp_lens_quadratic(text, table) -> Vec<u32>` (src/table.rs:348-361)
 * as called by SuffixTable::lcp_lens (src/table.rs:130-138):
 * lcp[0]=0, lcp[i]=|common byte prefix of suffix sa[i-1], suffix sa[i]|.
 * `sa` is checked to be a permutation of 0..n-1 (B200SA_ERR_BAD_ARG otherwise; the
 * reference would panic on an out-of-range index, src/table.rs:356-358). */
int b200sa_lcp(b200sa_ctx *ctx, const uint8_t *text, uint64_t n,
               const uint32_t *sa, uint32_t *lcp_out);

/* new + lcp_lens in one call; text and SA stay device-resident in between. */
int b200sa_build_lcp(b200sa_ctx *ctx, const uint8_t *text, uint64_t n,
                     uint32_t *sa_out, uint32_t *lcp_out);

/* ---- device-resident twins (PCIe-free; used by bench.py's `value`) ----
 * d_* are device pointers on the context's device; `stream` is a
 * cudaStream_t (NULL = the context's own stream).  The calls enqueue work and
 * synchronise the stream only where the pipeline must read sizes back. */
int b200sa_build_dev(b200sa_ctx *ctx, const uint8_t *d_text, uint64_t n,
                     uint32_t *d_sa, void *stream);
int b200sa_lcp_dev(b200sa_ctx *ctx, const uint8_t *d_text, uint64_t n,
                   const uint32_t *d_sa, uint32_t *d_lcp, void *stream);
/* new + lcp_lens in one device-resident call (the packed text of the build is
 * reused by the LCP kernels instead of being rebuilt). */
int b200sa_build_lcp_dev(b200sa_ctx *ctx, const uint8_t *d_text, uint64_t n,
                         uint32_t *d_sa, uint32_t *d_lcp, void *stream);

/* ---- batched queries over a device-resident index (SURVEY.md 8f-1) ----
 * Replaces SuffixTable::positions (src/table.rs:223-259) for a batch: query q
 * is bytes [q_off[q], q_off[q+1]) of d_queries; writes the SA range
 * [start[q], end[q]) whose entries are the match positions (SA order, as the
 * reference returns them). */
int b200sa_positions_dev(b200sa_ctx *ctx, const uint8_t *d_text, uint64_t n,
                         const uint32_t *d_sa, const uint8_t *d_queries,
                         const uint64_t *d_q_off, uint32_t nq,
                         uint32_t *d_start, uint32_t *d_end, void *stream);

/* ---- multi-GPU shards (SURVEY.md 8e; BASELINE config 5) ----
 * Type classification + LMS flags + (byte,type) histogram of ONE contiguous
 * shard text[lo,hi) of a longer text, one shard per GPU/process; the caller
 * (suffix_b200/sharded.py, torch.distributed over NCCL) exchanges the tiny
 * summaries between the two calls.  Replaces SuffixTypes::compute
 * (src/table.rs:592-615) and Bins::find_sizes (:686-704) for sharded input.
 *
 * 1. b200sa_shard_summary: *state_out = type of the shard's FIRST position as
 *    far as the shard (plus next_char = T[hi], or -1 at the end of the text)
 *    determines it: 0 Descending(L), 1 Ascending(S), 2 undetermined (every
 *    char up to and including next_char is equal).
 * 2. all-gather the states; tail_carry of shard r = first state != 2 among the
 *    shards after r.
 * 3. b200sa_shard_classify with prev_char = T[lo-1] (-1 for the first shard),
 *    next_char, tail_carry: S-type and LMS bitmaps (bit i&31 of word i>>5,
 *    shard-local positions), shard-local LMS positions (ascending), the
 *    768-bin histogram [0,256) L, [256,512) S-non-LMS, [512,768) LMS (host,
 *    u64, to be all-reduced) and the number of LMS positions.
 * d_shard must be 16-byte aligned. */
int b200sa_shard_summary(b200sa_ctx *ctx, const uint8_t *d_shard, uint64_t len, int next_char,
                         int *state_out, void *stream);
int b200sa_shard_classify(b200sa_ctx *ctx, const uint8_t *d_shard, uint64_t len, int prev_char, int next_char,
                          int tail_carry, uint32_t *d_stype_words, uint32_t *d_lms_words,
                          uint32_t *d_lmspos, uint64_t cap_lms, uint64_t *hist768, uint64_t *m_out, void *stream);

/* ---- generalized suffix array (SURVEY.md 8f-3; reference README.md:60-74, TODO:13-18) ----
 * The reference's own recipe: append the documents with a separator byte that occurs in none
 * of them, remember where each starts, build ONE SuffixTable, and map a match position back
 * to its document with a binary search.  This entry point does that mapping for a batch of
 * positions on the device: doc_starts[0..ndocs) ascending (doc_starts[0] = 0), a position p
 * belongs to the last document d with doc_starts[d] <= p; d_off = p - doc_starts[d].
 * (suffix_b200.GeneralizedSuffixTable is the host-side wrapper.) */
int b200sa_doc_ids_dev(b200sa_ctx *ctx, const uint32_t *d_pos, uint64_t count,
                       const uint32_t *d_doc_starts, uint32_t ndocs,
                       uint32_t *d_doc, uint32_t *d_off, void *stream);

/* ---- LCP-interval tree (SURVEY.md 8f-4; reference suffix_tree/src/lib.rs:392-505) ----
 * The internal nodes of the suffix tree the reference builds serially from SA + LCP are the
 * LCP intervals.  For every rank i: d_psv[i] = largest j < i with lcp[j] < lcp[i]
 * (0xFFFFFFFF if none), d_nsv[i] = smallest j > i with lcp[j] < lcp[i] (n if none); the
 * node that owns the boundary between suffixes i-1 and i is the interval
 * [psv[i], nsv[i]) of string depth lcp[i] (all-nearest-smaller-values over block minima). */
int b200sa_lcp_intervals_dev(b200sa_ctx *ctx, const uint32_t *d_lcp, uint64_t n,
                             uint32_t *d_psv, uint32_t *d_nsv, void *stream);

/* ---- suffix tree (SURVEY.md 8f-5; reference suffix_tree/src/lib.rs:392-505) ----
 * SuffixTree::from_suffix_table (:74-76) builds its tree with a serial insertion loop over
 * table() and lcp_lens() (to_suffix_tree, :392-505).  These entry points build the same tree
 * (structure, child order, string depths, label bytes, terminals) data-parallel from SA + LCP
 * and return it as arrays indexed by preorder id.  The reference's preorder is lexicographic
 * (children are keyed by the first byte of their label).  With lcp[n] := 0,
 * psv[i] = largest j < i with lcp[j] < lcp[i], nsv[i] = smallest j > i with lcp[j] < lcp[i] (or n),
 * pse[i] = largest j < i with lcp[j] <= lcp[i]:
 *   1. root: range [0, n), depth 0, parent 0xFFFFFFFF; its terminal is n (suffix_tree :84).
 *   2. internal nodes: one per boundary i in [1, n) with lcp[i] > 0 and pse[i] == psv[i];
 *      range [psv[i], nsv[i]), depth lcp[i].
 *   3. rank r is merged iff r+1 < n and lcp[r+1] == n - sa[r]: suffix sa[r] ends at the internal
 *      node of boundary r+1 (which keeps it as terminal and has children, :128-131, :432).  Every
 *      other rank r is a leaf: range [r, r+1), depth n - sa[r].
 *   4. preorder = ascending (sa_lo, depth); N = 1 + #internal + n - #merged <= 2n.
 *   5. parent of [lo, hi) (not the root): pd = max(lcp[lo], lcp[hi]); pd == 0: the root, else
 *      the node (plo, pd) with plo = lo if lcp[hi] > lcp[lo], else psv[lo].
 *   6. label = text[sa[lo] + pd, sa[lo] + depth); the node carries terminal sa[lo] iff
 *      depth == n - sa[lo].  (The reference's own label offsets of internal nodes depend on its
 *      insertion history, :474-480; the bytes are the same.)
 *   7. subtree_end = first[hi] (smallest id with sa_lo == hi) if hi < n, else N.
 *   8. children of v: v+1, then subtree_end of each child, while below subtree_end[v].
 * Every array of `out` holds at least `cap` entries; cap must be >= max(1, 2n).  On success
 * *num_nodes = N and entries [0, N) are written.  n = 0 gives the root alone (subtree_end 1).
 * Inputs are checked on the device (sa[r] < n, lcp[0] == 0, lcp[r] <= n - sa[r-1] and
 * <= n - sa[r], and every parent lookup finds its node): B200SA_ERR_BAD_ARG with a
 * b200sa_last_error detail otherwise.  Node ids are u32 with 0xFFFFFFFF reserved, so
 * n > B200SA_TREE_MAX_N returns B200SA_ERR_TOO_LARGE.  Device workspace is about 66 bytes per
 * text byte (the host entry point adds 56 for staging); B200SA_ERR_OOM if it cannot be had.
 * Measured on one H100 80GB HBM3 (400 W limit), device entry with the inputs and the six
 * arrays on the same card: n = 671,088,640 fits, n = 805,306,368 returns B200SA_ERR_OOM. */
#define B200SA_TREE_MAX_N 0x7FFFFFFFull
typedef struct {
    uint32_t *parent;       /* preorder id of the parent; 0xFFFFFFFF for the root (id 0)     */
    uint32_t *depth;        /* string depth (the reference's path_len)                       */
    uint32_t *sa_lo, *sa_hi;/* the subtree holds exactly the suffixes sa[sa_lo..sa_hi)       */
    uint32_t *label_start;  /* label = text[label_start, label_start + depth - depth[parent]) */
    uint32_t *subtree_end;  /* preorder id one past the node's last descendant               */
} b200sa_tree;
/* device buffers (sa, lcp in; the six arrays out); synchronises the stream before returning */
int b200sa_suffix_tree_dev(b200sa_ctx *ctx, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp,
                           const b200sa_tree *out, uint64_t cap, uint64_t *num_nodes, void *stream);
/* host buffers: SuffixTree::from_suffix_table(table) with sa = table(), lcp = lcp_lens() */
int b200sa_suffix_tree(b200sa_ctx *ctx, uint64_t n, const uint32_t *sa, const uint32_t *lcp,
                       const b200sa_tree *out, uint64_t cap, uint64_t *num_nodes);

/* ---- generalized suffix array without separators (SURVEY.md 8f-6; reference README.md:60-74, TODO:13-18) ----
 * Documents D_0 .. D_{k-1} (arbitrary bytes, possibly empty) are given as their concatenation C of
 * n = sum |D_d| bytes, with no separators, and doc_starts[d] = offset of D_d in C (ascending,
 * doc_starts[0] = 0, every entry <= n).  For a position p of document d, r_p = end_d - p and its
 * suffix is T_p = C[p, p + r_p).
 *   gsa   (the generalized suffix array G): all n positions sorted by (T_p, d).  Bytes compare
 *         lexicographically, a proper prefix sorts first, equal strings are ordered by document.
 *         This is the suffix array of D_0 $_0 D_1 $_1 ... with $_0 < $_1 < ... < every byte, without
 *         the terminator positions.  For k = 1 it is the SuffixTable of the single document.
 *   glcp  glcp[0] = 0, glcp[i] = common prefix length of T_{G[i-1]} and T_{G[i]} (never crosses a
 *         document end).  glcp_out / d_glcp may be NULL.
 * Built from SA and LCP of C (b200sa_build_lcp_dev): lo_i = the first rank sharing >= r_p bytes with
 * p = SA_C[i] (ranks with LCP_C[i] < r_p: i itself), G = the ranks sorted by (lo, r, d), and
 * glcp = min(r_a, r_b, min LCP_C over (lo_a, lo_b]) for neighbours a, b.  Only the ranks whose suffix
 * in C reaches past their document end are sorted.
 * B200SA_ERR_BAD_ARG with a b200sa_last_error detail when doc_starts does not start at 0, is not
 * ascending or has an entry above n, or when ndocs = 0 with n > 0 (the host entry checks on the host,
 * the device entry on the device); B200SA_ERR_TOO_LARGE above B200SA_MAX_N.  n = 0 and n = 1 return
 * without launching.  Device workspace, the SA + LCP build's included, measured on 100 MB on one
 * H100 80GB HBM3: about 46 bytes per text byte when few suffixes cross their document end (the build
 * alone holds 25), 78 when all do (n/4 copies of "ACGT"; the build alone 38); the host entry adds 9
 * for staging.  The phases report to b200sa_last_phase_times.  B200SA_DOCS_SORT2=1 forces the
 * two-stage sort (by document, then by (lo, r)) that keys of more than 64 bits take. */
int b200sa_docs_build(b200sa_ctx *ctx, const uint8_t *text, uint64_t n, const uint32_t *doc_starts, uint32_t ndocs,
                      uint32_t *gsa_out, uint32_t *glcp_out);
/* device buffers; synchronises the stream only to read the check word and the sort size back */
int b200sa_docs_build_dev(b200sa_ctx *ctx, const uint8_t *d_text, uint64_t n, const uint32_t *d_doc_starts,
                          uint32_t ndocs, uint32_t *d_gsa, uint32_t *d_glcp, void *stream);
/* Batched positions over G (b200sa_positions_dev with every suffix cut at its document end): query q is
 * bytes [q_off[q], q_off[q+1]) of d_queries (any bytes); writes the range [start[q], end[q]) of G whose
 * document suffixes start with it.  A match never crosses a document end.  d_gsa and d_doc_starts are
 * what b200sa_docs_build_dev was given and returned. */
int b200sa_docs_positions_dev(b200sa_ctx *ctx, const uint8_t *d_text, uint64_t n, const uint32_t *d_gsa,
                              const uint32_t *d_doc_starts, uint32_t ndocs, const uint8_t *d_queries,
                              const uint64_t *d_q_off, uint32_t nq, uint32_t *d_start, uint32_t *d_end, void *stream);

/* ---- generalized suffix tree with document counts (SURVEY.md 8f-7) ----
 * Documents D_0 .. D_{k-1} are given as for b200sa_docs_build: their concatenation C (n bytes) and
 * doc_starts.  For a position p of document d, len(p) = end_d - p and T_p = C[p, p + len(p)); G and
 * glcp are what b200sa_docs_build returns.
 * The tree is the compressed trie of the strings T_p.  Its nodes are the root, every distinct T_p,
 * and every string followed, among the T_p, by at least two distinct next bytes.  Children are
 * ordered by the first byte of their label and preorder is lexicographic, as for b200sa_suffix_tree.
 * The terminals of a node are all positions p whose T_p equals its string: a suffix that is a proper
 * prefix of another stays a terminal of a node with children (the reference's no-terminator
 * convention), and equal suffixes of different documents share one node.  The root has none.
 * As rules over (G, glcp), with len[r] = len(G[r]) and glcp[n] := 0: rules 1-8 of b200sa_suffix_tree,
 * with sa = G and lcp = glcp, except that
 *   3'. rank r is merged iff (r+1 < n and glcp[r+1] == len[r]) or (r > 0 and glcp[r] == len[r]); every
 *       other rank is a leaf with range [r, r+1) and depth len[r].  (For k = 1 the second condition never
 *       holds: the six arrays equal b200sa_suffix_tree's.)
 *   6.  label_start = G[lo] + pd as before; since depth <= len[lo], a label never crosses a document end.
 * and two more arrays per node v:
 *   term_end[v]   the terminals of v are G[sa_lo[v], term_end[v]) (== sa_lo[v] when there are none): a
 *                 prefix of the range, since proper prefixes sort first and equal strings are adjacent,
 *                 ordered by document;
 *   doc_count[v]  the number of distinct documents among G[sa_lo[v], sa_hi[v]); the root's is the number
 *                 of non-empty documents.
 * Inputs as for b200sa_suffix_tree (cap >= max(1, 2n), n <= B200SA_TREE_MAX_N, every array of `out` holds
 * cap entries) and b200sa_docs_build (doc_starts; the host entry checks it on the host, the device entry
 * on the device).  G and glcp are checked on the device with the tree's checks, glcp[r] bounded by the
 * len of both neighbours; every failure returns B200SA_ERR_BAD_ARG with a b200sa_last_error detail.
 * n = 0 gives the root alone (doc_count 0).  The phases report to b200sa_last_phase_times.  Device
 * workspace, measured on 100 MB on one H100 80GB HBM3: about 81 bytes per text byte (74 for n/4 copies
 * of "ACGT"); the caller's eight arrays add 64, G and glcp 8, and the host entry stages all of them.
 * (The output struct is b200sa_docs_tree_out: C gives a type and a function one namespace.) */
typedef struct {
    b200sa_tree tree;       /* rules 1-8 with 3' and document suffix lengths   */
    uint32_t *term_end;     /* terminals of v: G[sa_lo[v], term_end[v])        */
    uint32_t *doc_count;    /* distinct documents among G[sa_lo[v], sa_hi[v])  */
} b200sa_docs_tree_out;
/* device buffers (G, glcp, doc_starts in; the eight arrays out); synchronises the stream before returning */
int b200sa_docs_tree_dev(b200sa_ctx *ctx, uint64_t n, const uint32_t *d_gsa, const uint32_t *d_glcp,
                         const uint32_t *d_doc_starts, uint32_t ndocs, const b200sa_docs_tree_out *out,
                         uint64_t cap, uint64_t *num_nodes, void *stream);
/* host buffers */
int b200sa_docs_tree(b200sa_ctx *ctx, uint64_t n, const uint32_t *gsa, const uint32_t *glcp,
                     const uint32_t *doc_starts, uint32_t ndocs, const b200sa_docs_tree_out *out,
                     uint64_t cap, uint64_t *num_nodes);
/* Document frequency of a batch of ranges of G: d_start / d_end as b200sa_docs_positions_dev writes them.
 * d_count[q] = 0 for an empty range, else doc_count of a node whose range is [start[q], end[q]) (every node
 * with that range has the same count): the number of documents that contain query q.  A non-empty range
 * that is no node's returns B200SA_ERR_BAD_ARG.  The arrays are the first num_nodes entries of
 * b200sa_docs_tree_dev's sa_lo, sa_hi and doc_count.  Synchronises the stream. */
int b200sa_docs_tree_counts_dev(b200sa_ctx *ctx, const uint32_t *d_sa_lo, const uint32_t *d_sa_hi,
                                const uint32_t *d_doc_count, uint64_t num_nodes, const uint32_t *d_start,
                                const uint32_t *d_end, uint32_t nq, uint32_t *d_count, void *stream);

/* ---- document listing (SURVEY.md 8f-8) ----
 * Documents D_0 .. D_{k-1}, their concatenation C (n bytes), doc_starts, G and doc(p) as for
 * b200sa_docs_build.  Which documents contain a query, and how often, without the tree:
 *   byd   (n x u32) the ranks 0..n-1 sorted stably by (doc(G[r]), r).  Every position of document d has
 *         exactly one rank, so d's ranks are byd[doc_starts[d], doc_starts[d+1]) in increasing order.
 *   prev  (n x u32) for rank r of document d: prev[r] = r' + 1, where r' is the previous rank of d in
 *         byd, or 0 if r is d's first rank (the +1 keeps "none" below every threshold).
 * For a range [s, e) of G (b200sa_docs_positions_dev):
 *   listing  the ranks i in [s, e) with prev[i] <= s: the first rank of each document inside the range,
 *            so exactly one entry per distinct document of G[s, e), in ascending i (the table order of
 *            each document's first occurrence);
 *   docs     entry i reports d = doc(G[i]);
 *   tf       entry i optionally reports #{ranks of d in [s, e)}: the occurrences of the query in D_d
 *            (overlapping ones count, none crosses a document end).
 * b200sa_docs_list_index_dev writes byd and prev into caller buffers of n entries.  doc_starts is checked
 * on the device (B200SA_ERR_BAD_ARG with a b200sa_last_error detail, as b200sa_docs_tree_dev);
 * B200SA_ERR_TOO_LARGE above B200SA_MAX_N; n = 0 returns without launching.  Synchronises the stream
 * only to read the check word back.  Phases: docs_check, dlist_len, dlist_sort, dlist_prev. */
int b200sa_docs_list_index_dev(b200sa_ctx *ctx, uint64_t n, const uint32_t *d_gsa, const uint32_t *d_doc_starts,
                               uint32_t ndocs, uint32_t *d_byd, uint32_t *d_prev, void *stream);
/* Document listing of a batch of ranges d_start / d_end of G.  Always writes d_offsets (nq + 1 x u64,
 * exclusive: query q's entries are [offsets[q], offsets[q+1])) and *total = offsets[nq].  Writes
 * d_docs[offsets[q], offsets[q+1]) and, if d_tf is non-NULL, d_tf at the same places, only when
 * total <= cap; otherwise it returns B200SA_OK with nothing written past the offsets, so that the caller
 * can size the buffers and call again.  cap = 0 (d_docs may then be NULL) is the document-frequency
 * query: offsets[q+1] - offsets[q] is the number of documents that contain query q.  byd and prev must
 * be what b200sa_docs_list_index_dev wrote for the same G and doc_starts; they are not verified.  A range
 * with start > end or end > n returns B200SA_ERR_BAD_ARG (checked on the device).  Block minima over
 * prev are rebuilt on every call (one read of 4n bytes); device workspace besides them is 12 bytes per
 * chunk of 1024 ranks of every range plus 8 per query.  Synchronises the stream (it reads the chunk
 * count and the total back).  Phases: dlist_levels, dlist_count, dlist_scan, dlist_emit. */
int b200sa_docs_list_dev(b200sa_ctx *ctx, uint64_t n, const uint32_t *d_gsa, const uint32_t *d_doc_starts,
                         uint32_t ndocs, const uint32_t *d_byd, const uint32_t *d_prev, const uint32_t *d_start,
                         const uint32_t *d_end, uint32_t nq, uint64_t *d_offsets, uint32_t *d_docs, uint32_t *d_tf,
                         uint64_t cap, uint64_t *total, void *stream);

/* ---- top-k document retrieval (SURVEY.md 8f-9) ----
 * For a range [s, e) of G the listing above gives one entry (d, tf) per distinct document.  Then
 *   key(d, tf)   orders entries by tf descending, then d ascending (((u64)tf << 32) | (0xFFFFFFFF - d),
 *                largest first); documents are distinct within a query, so the order is total;
 *   top_k(s, e)  the min(k, df) entries with the largest keys, in key order;
 * an empty range (s = e: b"" or an absent query) has no entries.
 * b200sa_docs_topk_dev writes d_count[q] = min(k, df(q)) and, for j < d_count[q], d_docs[q*k + j] and
 * d_tf[q*k + j]: query q's top-k in key order.  Slots j >= d_count[q] are not written.  Arguments as for
 * b200sa_docs_list_dev (byd and prev are not verified; a range with start > end or end > n returns
 * B200SA_ERR_BAD_ARG, checked on the device); k = 0 or k > B200SA_TOPK_MAX returns B200SA_ERR_BAD_ARG
 * (one block sorts the survivors of a query in shared memory; for larger k list with
 * b200sa_docs_list_dev); nq = 0 returns without launching; n = 0 gives all counts 0.
 * The listing is materialised in rounds: runs of consecutive queries whose entries fit
 * B200SA_TOPK_ROUND_ENTRIES (a larger query, at most ndocs entries, is a round of its own); more than
 * one round reads the per-query offsets back.  Device workspace: the listing's (block minima, 12 bytes per
 * chunk of 1024 ranks of every range) plus 20 bytes per query and 16 bytes per entry of the largest round;
 * with more than one round, 8 more per query and per chunk of that round.  Synchronises the stream.
 * Phases: dlist_levels, dlist_count, dlist_scan, then per round topk_emit, topk_select. */
#define B200SA_TOPK_MAX 1024
#define B200SA_TOPK_ROUND_ENTRIES (1ull << 26)
int b200sa_docs_topk_dev(b200sa_ctx *ctx, uint64_t n, const uint32_t *d_gsa, const uint32_t *d_doc_starts,
                         uint32_t ndocs, const uint32_t *d_byd, const uint32_t *d_prev, const uint32_t *d_start,
                         const uint32_t *d_end, uint32_t nq, uint32_t k, uint32_t *d_count, uint32_t *d_docs,
                         uint32_t *d_tf, void *stream);

/* ---- matching statistics and super-maximal exact matches (DESIGN.md 6b f-10) ----
 * Index: a text T of n bytes with sa and lcp as b200sa_build_lcp_dev returns them, or the documents'
 * concatenation C with G, glcp and doc_starts as b200sa_docs_build_dev takes and returns them.  S_p is the
 * suffix at p: T[p, n), or C[p, end of p's document).  A string occurs if it is a prefix of some S_p; with
 * documents an occurrence never crosses a document end.
 * Queries as for b200sa_positions_dev: query q is bytes [q_off[q], q_off[q+1]) of d_queries, and
 * q_bytes = q_off[nq] is passed by the caller, so that no read-back is needed to size the launch.  A pattern
 * position is a byte index x in [0, q_bytes); it lies in query q(x), whose end is E(x) = q_off[q(x)+1].
 * For every pattern position x:
 *   len[x]              the largest l <= E(x) - x such that queries[x, x+l) occurs: a match never runs past
 *                       the end of its own query;
 *   [start[x], end[x])  the range of the table (sa or G) whose suffixes start with queries[x, x+len[x]):
 *                       what b200sa_positions_dev / b200sa_docs_positions_dev return for that string when
 *                       len[x] > 0, and (0, 0) when len[x] = 0 (b"" matches nothing).
 * d_len, d_start and d_end hold q_bytes u32 each.  d_start and d_end are both given or both NULL; without
 * them only len is written, d_lcp / d_glcp may be NULL and no block minima are built.  One binary search
 * per position carries the common-prefix lengths of its two bounds, so it ends with the longest match and
 * a rank that attains it; the range is the LCP interval of depth len[x] around that rank.  Block minima
 * over lcp are rebuilt on every call (one read of 4n bytes).
 * sa and lcp (G and glcp) must be what the build returned; they are not verified.  q_off is checked on the
 * device (q_off[0] = 0, ascending, q_off[nq] = q_bytes), and so is doc_starts by the documents entry:
 * B200SA_ERR_BAD_ARG with a b200sa_last_error detail, as for a required NULL pointer.  n or q_bytes above
 * B200SA_MAX_N returns B200SA_ERR_TOO_LARGE.  nq = 0 or q_bytes = 0 return without launching; n = 0 gives
 * len = start = end = 0 everywhere.  No byte outside [d_text, d_text + n) and [d_queries, d_queries + q_bytes)
 * is read: the buffers need no padding and no alignment.  Synchronises the stream only to read the check
 * words back.  Phases: match_check, match_levels (with ranges), match_search. */
int b200sa_match_stats_dev(b200sa_ctx *ctx, const uint8_t *d_text, uint64_t n, const uint32_t *d_sa,
                           const uint32_t *d_lcp, const uint8_t *d_queries, const uint64_t *d_q_off,
                           uint32_t nq, uint64_t q_bytes, uint32_t *d_len, uint32_t *d_start,
                           uint32_t *d_end, void *stream);
int b200sa_docs_match_stats_dev(b200sa_ctx *ctx, const uint8_t *d_text, uint64_t n, const uint32_t *d_gsa,
                                const uint32_t *d_glcp, const uint32_t *d_doc_starts, uint32_t ndocs,
                                const uint8_t *d_queries, const uint64_t *d_q_off, uint32_t nq,
                                uint64_t q_bytes, uint32_t *d_len, uint32_t *d_start, uint32_t *d_end,
                                void *stream);
/* Super-maximal exact matches (SMEMs) of query q at threshold min_len >= 1: the positions x of q with
 * len[x] >= min_len and (x = q_off[q] or len[x-1] <= len[x]).  Dropping the first byte of a match leaves a
 * match, so len[x+1] >= len[x] - 1 and x + len[x] never decreases inside a query; hence a match
 * [x, x+len[x]) lies inside another match of the query exactly when x-1 is in the query and
 * len[x-1] > len[x], and the SMEMs are the matches of at least min_len bytes contained in no other.
 * d_len is what the calls above wrote for the same q_off.  Follows the listing's protocol: always writes
 * d_offsets (nq + 1 x u64, exclusive: query q's SMEMs are [offsets[q], offsets[q+1])) and
 * *total = offsets[nq]; writes d_qpos[0, total), the offset x - q_off[q] of each SMEM inside its query, in
 * ascending x, only when total <= cap; cap = 0 (d_qpos may then be NULL) counts only.  The caller gathers
 * len / start / end at q_off[q] + qpos.  min_len = 0 returns B200SA_ERR_BAD_ARG; q_off is checked as above;
 * q_bytes above B200SA_MAX_N returns B200SA_ERR_TOO_LARGE; nq = 0 writes offsets[0] = 0.  Device workspace:
 * 8 bytes per query byte.  Synchronises the stream (it reads the total back).  Phases: match_check,
 * smem_flag, smem_scan, smem_emit. */
int b200sa_smems_dev(b200sa_ctx *ctx, const uint64_t *d_q_off, uint32_t nq, uint64_t q_bytes,
                     const uint32_t *d_len, uint32_t min_len, uint64_t *d_offsets, uint32_t *d_qpos,
                     uint64_t cap, uint64_t *total, void *stream);

/* ---- repeats: what in the text repeats itself (DESIGN.md 6b f-11) ----
 * Index as for the matching statistics: a text T of n bytes with sa and lcp, or the concatenation C with G,
 * glcp and doc_starts (pass G as d_sa and glcp as d_lcp).  R is the table, lam its LCP array with
 * lam[n] := 0, S_p the suffix at p cut at the end of p's document, len(p) = |S_p|, ds(p) and de(p) the start
 * and end of p's document (0 and n for a single text).  L = min_len >= 1.  The gram at p is S_p[0, L),
 * defined when len(p) >= L; it never crosses a document end.
 * 1. Repeat length.  rl[p] = max(lam[r], lam[r+1]) for the rank r with R[r] = p: the largest l such that
 *    S_p[0, l) is a prefix of S_p' for some p' != p.  rl[p] >= L iff the gram at p occurs elsewhere.
 * 2. Runs at L.  The maximal rank ranges [a, b), b - a >= 2, with lam[i] >= L for a < i < b.  They
 *    correspond one to one to the distinct strings of L bytes that occur at least twice, and [a, b) is the
 *    range b200sa_positions_dev / b200sa_docs_positions_dev return for that string.  first(run) = min R[a..b),
 *    last(run) = max R[a..b).  Positions are ordered by document, so first lies in the run's lowest document
 *    and last in its highest.
 * 3. Flagged positions, by mode (a position outside every run is never flagged):
 *      B200SA_REPEAT_ANY          p is in a run: the gram at p occurs at another position;
 *      B200SA_REPEAT_EARLIER      p != first(run): it occurs at a smaller position;
 *      B200SA_REPEAT_OTHER_DOC    first(run) < ds(p) or last(run) >= de(p): it occurs in a different document;
 *      B200SA_REPEAT_EARLIER_DOC  first(run) < ds(p): it occurs in a document of smaller index.
 *    For a single text the two document modes flag nothing by definition and are rejected.
 * 4. Duplicate spans.  Byte x is covered iff some flagged p has p <= x < p + L.  The spans are the maximal
 *    intervals [begin, end) of covered bytes with no document start strictly inside: touching intervals of
 *    one document merge, those of adjacent documents do not.  Each span lies in one document and is at
 *    least L bytes long.  Spans are reported by ascending begin, in coordinates of the concatenation;
 *    covered = the number of covered bytes = the sum of end - begin.
 * The two counting calls follow the listing's protocol: *total (and *covered) are always written; the arrays
 * are written only when total <= cap, and never past total; cap = 0 (the arrays may then be NULL) counts only.
 * min_len = 0, an unknown mode, a document mode without doc_starts or a required NULL pointer return
 * B200SA_ERR_BAD_ARG with a b200sa_last_error detail; doc_starts is checked on the device; n above
 * B200SA_MAX_N returns B200SA_ERR_TOO_LARGE; n = 0 gives totals 0 without launching; min_len > n is legal and
 * gives nothing.  sa and lcp must be what the build returned; they are not verified.  The counting calls
 * synchronise the stream (they read the totals back).  Device workspace per text byte: runs 0, with
 * first / last 8 or 12; spans 4.25 for ANY, 8.25 for EARLIER and EARLIER_DOC, 12.25 for OTHER_DOC. */
enum {
    B200SA_REPEAT_ANY = 0,
    B200SA_REPEAT_EARLIER = 1,
    B200SA_REPEAT_OTHER_DOC = 2,
    B200SA_REPEAT_EARLIER_DOC = 3
};
/* rl in text order: d_rl[p], n x u32.  Phase: rep_lens. */
int b200sa_repeat_lens_dev(b200sa_ctx *ctx, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp,
                           uint32_t *d_rl, void *stream);
/* The runs at min_len, ascending: d_start[i], d_end[i] and, where non-NULL, d_first[i], d_last[i].
 * Phases: rep_count, rep_segments (with first / last), rep_emit. */
int b200sa_repeat_runs_dev(b200sa_ctx *ctx, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp,
                           uint32_t min_len, uint32_t *d_start, uint32_t *d_end, uint32_t *d_first,
                           uint32_t *d_last, uint64_t cap, uint64_t *total, void *stream);
/* The spans for `mode`.  d_doc_starts = NULL with ndocs = 0: a single text.  Phases: rep_check (with
 * documents), rep_segments (every mode but ANY), rep_flag, rep_cover, rep_count, rep_emit. */
int b200sa_duplicate_spans_dev(b200sa_ctx *ctx, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp,
                               const uint32_t *d_doc_starts, uint32_t ndocs, uint32_t min_len, int mode,
                               uint32_t *d_begin, uint32_t *d_end, uint64_t cap, uint64_t *total,
                               uint64_t *covered, void *stream);

/* ---- longest previous factor and LZ77 factorization (DESIGN.md 6b f-12) ----
 * Index as for the repeats: R the table (sa, or G for documents: pass G as d_sa and glcp as d_lcp), lam its
 * LCP array, S_p the suffix at p cut at the end of p's document, positions in coordinates of the text or
 * of the concatenation, R[r] = p.  No doc_starts is needed: glcp never crosses a document end.
 * 1. Nearest smaller positions.  psv(r) = the largest r' < r with R[r'] < p, nsv(r) = the smallest r' > r
 *    with R[r'] < p; either may be absent.  lcp(a, b) = min lam(a, b] for ranks a < b; lL = lcp(psv, r),
 *    lR = lcp(r, nsv), a missing side counting 0.
 * 2. LPF.  lpf[p] = max(lL, lR): the largest l such that S_p[0, l) is a prefix of S_q for some q < p;
 *    the occurrence may overlap p (q + l > p).  (Crochemore & Ilie, IPL 2008.)
 * 3. Source.  src[p] = R[psv] if lL >= lR and lL > 0, else R[nsv] if lR > 0, else B200SA_LZ_LITERAL.
 *    The tie goes to the psv side.  src[p] is AN earlier occurrence of S_p[0, lpf[p]), not necessarily the
 *    leftmost or the closest one.
 * 4. Factorization.  next(p) = p + max(1, lpf[p]); the factor starts are f_0 = 0 and f_(i+1) = next(f_i)
 *    while below n.  Factor i is (start = f_i, len = max(1, lpf[f_i]), src = src[f_i]); a literal has
 *    len = 1 and src = B200SA_LZ_LITERAL, its byte is the text's byte at start.  z = the number of factors.
 * Properties: lpf[p+1] >= lpf[p] - 1, so next never decreases and next(p) > p; with documents
 * lpf[p] <= de(p) - p, so no factor crosses a document end and every non-empty document starts a factor:
 * the document call is the single-text call applied to G and glcp.
 * b200sa_lz77_dev follows the listing's protocol: *total = z is always written; the arrays are written only
 * when z <= cap, and never past z; cap = 0 (the arrays may then be NULL) counts only.  A required NULL
 * pointer returns B200SA_ERR_BAD_ARG; n above B200SA_MAX_N returns B200SA_ERR_TOO_LARGE; n = 0 gives z = 0
 * without launching.  sa and lcp must be what the build returned; they are not verified.  The
 * factorization synchronises the stream (it reads z back) and leaves the number of parse rounds,
 * ceil(log2 z), in b200sa_last_stats().doubling_rounds.  Device workspace per text byte (computed, not
 * measured): lpf 0.26 (two sets of 32-ary block minima); lz77 16.4 (lpf, src, two jump arrays, a 1-bit
 * mark and the minima). */
#define B200SA_LZ_LITERAL 0xFFFFFFFFu
/* lpf and (when d_src != NULL) src in text order, n x u32 each.  Phases: lz_levels, lz_lpf. */
int b200sa_lpf_dev(b200sa_ctx *ctx, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp, uint32_t *d_lpf,
                   uint32_t *d_src, void *stream);
/* The factors by ascending start.  Phases: lz_levels, lz_lpf, lz_parse, lz_count, lz_emit. */
int b200sa_lz77_dev(b200sa_ctx *ctx, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp, uint32_t *d_start,
                    uint32_t *d_len, uint32_t *d_src, uint64_t cap, uint64_t *total, void *stream);

/* ---- Burrows-Wheeler transform and its inverse (DESIGN.md 6b f-13) ----
 * Documents D_0 .. D_(k-1), k >= 1, with concatenation C (n bytes) and doc_starts as b200sa_docs_build takes
 * them; empty documents are allowed.  A single text is k = 1, doc_starts = [0], G = SA.
 * 1. Rows.  There are n + k rows.  Row d < k is the rotation $_d D_d.  Row k + r is the rotation that starts
 *    at position G[r] of its document d: C[G[r], end_d) $_d D_d[0, G[r] - start_d).  The terminators order
 *    as $_0 < $_1 < ... < every byte: G's order with the k terminator rows placed first.
 * 2. L.  L[d] is the last byte of D_d, or $_d when D_d is empty.  L[k + r] is C[G[r] - 1], or $_d when G[r]
 *    is the start of its document d (with several empty documents at one offset, the last one owns it).
 * 3. Output.  bwt = the n bytes of L in row order with the k terminators removed; term_rows[d] = the row
 *    whose L is $_d (distinct, not sorted by d).  For a single text term_rows[0] is the primary index,
 *    1 + the rank of position 0.
 * 4. Runs.  r = the number of maximal runs of equal symbols in the full L of n + k symbols; every
 *    terminator is a symbol of its own.
 * 5. Inverse.  psi(d) = term_rows[d] for d < k; the non-terminator rows of L, stably sorted by byte: the
 *    j-th is psi(k + j) and its byte is F[k + j].  Document d is the bytes F along psi from row d, until the
 *    walk returns to a row below k.
 * 6. Validity.  (bwt, term_rows) is the image of some documents exactly when the term rows are in range
 *    and distinct, and following psi from every row d < k returns to d without meeting another row below
 *    k, these k cycles covering all n + k rows.
 * A required NULL pointer, doc_starts that fails the b200sa_docs_build checks (checked on the device),
 * d_doc_starts with ndocs = 0 and n > 0, and on the inverse ndocs = 0, term rows out of range or repeated or
 * an input that breaks the validity rule return B200SA_ERR_BAD_ARG with a b200sa_last_error detail; the
 * inverse then writes no byte and no start.  n + k above B200SA_MAX_N returns B200SA_ERR_TOO_LARGE before
 * any launch.  n = 0 writes the k term rows and no bytes.  sa / G must be what the build returned; they are
 * not verified.  The inverse ranks psi with rulers: the rows below k and rows picked by a hash of the row
 * index, one in s (B200SA_BWT_RULER, default 64; a spacing above n leaves the terminator rows alone); it
 * leaves its pointer-doubling rounds in b200sa_last_stats().doubling_rounds.  Device workspace per text
 * byte (computed from the buffers, not measured): forward 1.13 (L bytes and a 1-bit terminator flag);
 * inverse 20.25 + at most 28 / s (sorted bytes and indices and the sort's key copy 12, psi and F 8, the ruler bitmap
 * and its prefix 0.25; per ruler its row, walk length and two list entries), plus 16 per document. */
/* d_doc_starts = NULL with ndocs = 0: a single text (k = 1).  d_sa is SA, or G for documents.  runs may be
 * NULL; if it is not, the call reads r back and synchronises.  Writes d_bwt (n bytes) and d_term_rows (k).
 * Phases: bwt_check (with documents), bwt_gather, bwt_compact. */
int b200sa_bwt_dev(b200sa_ctx *ctx, uint64_t n, const uint8_t *d_text, const uint32_t *d_sa,
                   const uint32_t *d_doc_starts, uint32_t ndocs, uint8_t *d_bwt, uint32_t *d_term_rows,
                   uint64_t *runs, void *stream);
/* k = ndocs >= 1.  Writes C (n bytes) and, when d_doc_starts_out != NULL, doc_starts (k entries).
 * Synchronises: it reads the validity word back.  Phases: unbwt_sort, unbwt_walk, unbwt_rank, unbwt_emit. */
int b200sa_unbwt_dev(b200sa_ctx *ctx, uint64_t n, uint32_t ndocs, const uint8_t *d_bwt,
                     const uint32_t *d_term_rows, uint8_t *d_text_out, uint32_t *d_doc_starts_out, void *stream);

/* ---- approximate positions: occurrences with at most k mismatches (DESIGN.md 6b f-14) ----
 * Index: a text T of n bytes with its sa, or the documents' concatenation C with G and doc_starts as
 * b200sa_docs_build_dev takes and returns them.  No LCP array is needed.  end(p) = n for a single text, or
 * the end of p's document.  Query q is bytes [q_off[q], q_off[q+1]) of d_queries, m bytes of any values.
 * One threshold k, 0 <= k <= B200SA_APPROX_MAX_K, holds for the whole call.
 * An occurrence of q is a position p with
 *   1. p + m <= end(p): the window never crosses the text end or a document end;
 *   2. mis(p) = #{x < m : T[p+x] != q[x]} <= k.
 * m = 0 has no occurrences (b"" matches nothing, as for b200sa_positions_dev).  When 0 < m <= k every window
 * of m bytes is an occurrence.  For k = 0 the occurrences are the positions of table[start, end) that
 * b200sa_positions_dev / b200sa_docs_positions_dev return, in ascending order.
 * Output follows the listing's protocol: d_offsets (nq + 1 x u64, exclusive) and *total = offsets[nq] are
 * always written; d_pos[offsets[q], offsets[q+1]) holds query q's occurrences in ascending p, and
 * d_mismatches (may be NULL) mis(p) beside them, written only when total <= cap and never past total.
 * cap = 0 (d_pos may then be NULL) counts only.
 * Method: pigeonhole filter and verification.  When m > k the query is cut into k + 1 pieces,
 * piece j = [j*m/(k+1), (j+1)*m/(k+1)); a window with at most k mismatches matches some piece exactly.  Each
 * rank of the table range of piece j is a candidate, verified against the other pieces; it is reported only
 * when no piece before j matches exactly, so every occurrence is reported once, by its first exact piece.
 * A required NULL pointer, k > B200SA_APPROX_MAX_K, a bad q_off (q_off[0] != 0 or not ascending; checked on
 * the device, q_off[nq] is read back as the queries' length) and, for documents, doc_starts that fails the
 * b200sa_docs_build checks (on the device) or ndocs = 0 with n > 0 return B200SA_ERR_BAD_ARG with a
 * b200sa_last_error detail.  n or q_off[nq] above B200SA_MAX_N, or nq * (k + 1) >= 2^32 - 1, return
 * B200SA_ERR_TOO_LARGE.  nq = 0 writes offsets[0] = 0 and total = 0; n = 0 gives empty lists without launching
 * a search kernel.  sa / G must be what the build returned; they are not verified.  No byte outside
 * [d_text, d_text + n) and [d_queries, d_queries + q_off[nq]) is read: the buffers need no padding and no
 * alignment.  Synchronises the stream (it reads the total back).  Device workspace (computed from the
 * buffers, not measured): 16 bytes per piece (nq * (k + 1) pieces), 12 bytes per candidate chunk (1024 ranks
 * of a piece's range, or of the whole table for a query of 0 < m <= k), and, when the occurrences are
 * fetched, 24 bytes per output entry plus the radix sort's tile status (at most 1 byte per entry).
 * B200SA_ERR_OOM when that cannot be allocated.  Phases: approx_check, approx_pieces, approx_scan,
 * approx_count, approx_emit, approx_sort (the last two only when total <= cap and total > 0).
 *
 * ---- the edit metric: occurrences within k insertions, deletions and substitutions (DESIGN.md 6b f-15) ----
 * The k argument is threshold | flags: threshold = k & 0xFFFF, 0 <= threshold <= B200SA_APPROX_MAX_K, and the
 * only flag is B200SA_APPROX_EDIT.  Without the flag the call is the Hamming search above, bit for bit.  Other
 * flag bits, or a threshold above B200SA_APPROX_MAX_K, return B200SA_ERR_BAD_ARG with a b200sa_last_error detail
 * that names B200SA_APPROX_MAX_K; the TOO_LARGE slot check counts nq * (threshold + 1).
 * With B200SA_APPROX_EDIT (k below meaning the threshold): index, queries and end(p) are as above.  ED is the
 * Levenshtein distance, unit cost for each substitution, insertion and deletion.  For a position p in [0, n):
 *   dist(p) = min over e with p <= e <= end(p) of ED(q, T[p, e)),
 * the best alignment of the whole query that starts at p and crosses neither the text end nor a document end;
 * the empty substring (e = p) counts.  p is an occurrence iff dist(p) <= k.  Occurrences are listed by ascending
 * p with dist(p) in d_mismatches (may be NULL) beside them; offsets, total, cap, ordering, workspace and phase
 * names are as above.  m = 0 has no occurrences; 0 < m <= k makes every position an occurrence (dist <= m).
 * k = 0 gives exactly the set b200sa_positions_dev returns.  For every k the Hamming occurrences are a subset of
 * the edit occurrences, with dist(p) <= mis(p) on them.  One locus yields a run of neighbouring starts (an exact
 * hit at p also puts p - 1 and p + 1 at distance 1, when they lie in p's document); no filtering is applied
 * (B200SA_APPROX_LOCI, f-23 below, keeps one hit per locus).
 * Method: the same pieces and slots.  A candidate s of piece j (offset o_j) considers the starts p of s's
 * document with |p - (s - o_j)| <= k and computes their dist(p) by one banded reversed Sellers DP over the
 * diagonals [s - o_j - 2k, s - o_j + 2k].  It emits p iff dist(p) <= k and it is the least (i, s'') such that
 * piece i occurs exactly at s'' inside p's document with |s'' - o_i - p| <= k; every occurrence has one such
 * least pair (the partition lemma), so each is emitted once.  A query of 0 < m <= k keeps the whole-table slot
 * and each rank s reports itself.
 *
 * ---- best hits: each query's occurrences at its least distance, plus a slack (DESIGN.md 6b f-16) ----
 * With B200SA_APPROX_BEST the k argument is threshold | B200SA_APPROX_SLACK(s) | B200SA_APPROX_BEST, optionally
 * | B200SA_APPROX_EDIT: threshold = k & 0xFF and s = (k >> 8) & 0xFF, both at most B200SA_APPROX_MAX_K; any other
 * bit, or a threshold or s above it, returns B200SA_ERR_BAD_ARG with a detail that names B200SA_APPROX_MAX_K.
 * Without B200SA_APPROX_BEST, k is decoded as above (bits 8-15 are threshold bits) and nothing changes.
 * d(p) is mis(p), or dist(p) with B200SA_APPROX_EDIT.  The occurrences of q at a threshold t are what the call
 * without B200SA_APPROX_BEST returns at t; best(q) is the least d(p) over q's occurrences at the threshold,
 * undefined when it has none.  Query q lists its occurrences with d(p) <= t(q), t(q) = min(threshold,
 * best(q) + s): q's list is exactly what the call without the flag returns for q at threshold t(q), by ascending
 * p with d(p) in d_mismatches.  A query with no occurrence within the threshold lists nothing.  So s = 0 lists
 * the best stratum (every listed d equals best(q)); s >= threshold gives the call without the flag at threshold,
 * bit for bit; threshold = 0 gives the exact call.  Offsets, total, cap, the nq * (threshold + 1) TOO_LARGE
 * check, nq = 0, n = 0, m = 0 and the bytes read are as above.
 * Method: rounds t = 0, 1, .., threshold.  Round t searches, with the pieces and verification above at
 * threshold t, the live queries: those with no occurrence in an earlier round, and those whose first round
 * with an occurrence, best(q), has t <= best(q) + s.  The search runs on the live queries compacted into a
 * batch of their own.  The rounds stop when no query is live; b200sa_last_stats().doubling_rounds holds the
 * number run.  q's count is its count in its last live round.  When total <= cap, one emission at each distinct
 * t(q) over the queries that end there writes their lists into place.  Device workspace (computed, not
 * measured): 25 bytes per query and 1 per query byte for the batches, plus what the search above takes per
 * round for its batch at threshold t (16 bytes per piece, 12 per candidate chunk), and, when fetched, 24 bytes
 * per entry of the largest group plus the sort's tile status.  Phases: approx_check; per round best_compact,
 * approx_pieces, approx_scan, approx_count, best_update; per emitted group best_compact, approx_pieces,
 * approx_scan, approx_count, approx_emit, approx_sort, best_scatter.
 *
 * ---- IUPAC nucleotide codes in the queries (DESIGN.md 6b f-17) ----
 * With B200SA_APPROX_IUPAC (bit 24) in k, each query byte is an IUPAC code that stands for a class of text bytes:
 * A C G T for themselves, U for T, R = AG, Y = CT, S = CG, W = AT, K = GT, M = AC, B = CGT, D = AGT, H = ACT,
 * V = ACG, N = ACGT, in either case.  Any other query byte ('-' and '.' included) returns B200SA_ERR_BAD_ARG,
 * checked on the device in phase approx_check, with a detail that names the byte and its offset in d_queries.
 * The flag combines with B200SA_APPROX_EDIT, with B200SA_APPROX_BEST | B200SA_APPROX_SLACK(s), or with both;
 * the threshold is decoded as above (k & 0xFFFF, or k & 0xFF with B200SA_APPROX_BEST).  Without it nothing changes.
 * Text side: only the uppercase bytes A C G T are in any class, and nothing is folded.  Lowercase (soft-masked)
 * bases, N, U and every other text byte match no query symbol and count as a mismatch; uppercase a soft-masked
 * text before building the table.  (The filter looks up exact pieces in the table, so a case-insensitive or
 * U = T text would need 2^len variants of each piece.)
 * Definitions: those above with "T[p + x] != q[x]" read as "T[p + x] is not in the class of q[x]": mis(p) counts
 * such positions, and in dist(p) a substitution costs 0 iff the text byte is in the class.  best(q), t(q), the
 * window and document-end rules, offsets, ordering, cap, the nq * (threshold + 1) TOO_LARGE check, m = 0 and
 * n = 0 are as above.  So a query of uppercase A C G T alone gives exactly the call without the flag (positions
 * and distances, either metric, with or without best); lowercase letters act as their uppercase, U as T; and at
 * threshold 0 the Hamming list is the sorted union of b200sa_positions_dev over the query's concrete expansions.
 * Method: A C G T U are the concrete symbols (classes of one base); the maximal runs of concrete symbols are the
 * query's stretches, of lengths L_i, and P = threshold + 1.  t is the largest length with sum floor(L_i / t) >= P;
 * stretch i, left to right, gives c_i = min(floor(L_i / t), pieces still needed) pieces, piece j of the stretch
 * being [j*L_i/c_i, (j+1)*L_i/c_i) from its start.  The pieces are disjoint, concrete and at least t long, so
 * each is one exact range of the table; for a concrete query they are the pieces above.  If sum L_i < P (m <=
 * threshold included) the query keeps the whole-table slot: every rank is a candidate, verified in full.  The
 * reporter rules above carry over with each piece's offset and length from a per-slot table: the partition lemma
 * needs only threshold + 1 disjoint pieces, not a cover, so each occurrence is still reported once.  Device
 * workspace (computed, not measured): what the call takes without the flag, plus 1 byte per query byte for the
 * canonical copy and 8 bytes per slot for the piece table.
 *
 * ---- both DNA strands (DESIGN.md 6b f-18) ----
 * With B200SA_APPROX_BOTH_STRANDS (bit 28) in k, each query is also searched as its reverse complement, and q
 * gets one list over both strands.  The flag combines with B200SA_APPROX_EDIT, with B200SA_APPROX_BEST |
 * B200SA_APPROX_SLACK(s), with B200SA_APPROX_IUPAC, or with any mix of them; the threshold is decoded as above.
 * Without it nothing changes.  comp swaps A <-> T, C <-> G, a <-> t and c <-> g, and every other byte (U
 * included) is its own complement.  With B200SA_APPROX_IUPAC the class of comp(x) is the set of the complements
 * of x's class: A <-> T, C <-> G, U -> A, R <-> Y, K <-> M, B <-> V, D <-> H, and S, W, N themselves, in either
 * case; the byte check runs first, on d_queries, and its detail names the offset there.  rc(q)[x] =
 * comp(q[m - 1 - x]).  A minus-strand occurrence of q at p is an occurrence of rc(q) at p under the call's metric,
 * threshold and IUPAC setting, with d(p) the distance computed for rc(q): p is the leftmost text position of the
 * window or alignment, and the window and document-end rules are as above.  q's list is the union of (p, +) over
 * q's occurrences and (p, -) over rc(q)'s, ordered by (p, strand) with + first; d_mismatches[i] = d(p) |
 * (minus ? B200SA_APPROX_MINUS : 0), and with d_mismatches = NULL one p can appear twice.  Offsets and total
 * count both strands.  With B200SA_APPROX_BEST, best(q) is the least d over both strands, t(q) = min(threshold,
 * best(q) + s), and q lists both strands' occurrences at t(q).  So the + entries are exactly the call without the
 * flag on q (at t(q) with B200SA_APPROX_BEST), the - entries exactly that call on rc(q) with bit 31 set, a
 * palindrome (rc(q) = q) lists each occurrence twice, m = 0 lists nothing and 0 < m <= threshold lists every
 * window twice.  q_off[nq] above B200SA_MAX_N / 2, or 2 * nq * (threshold + 1) >= 2^32 - 1, returns
 * B200SA_ERR_TOO_LARGE in phase approx_check, before any kernel reads the queries.
 * Method: a doubled batch, entry 2q = q and entry 2q + 1 = rc(q) (built from the canonical copy with
 * B200SA_APPROX_IUPAC), is searched as 2 nq queries; its sorted (entry, p) keys are merged per query by a binary
 * search in the other strand's sublist.  With B200SA_APPROX_BEST a query and its reverse complement are live as
 * a pair with one best.  Device workspace (computed, not measured): 2 bytes per query byte and 32 per query for
 * the doubled batch and its offsets, plus what the search takes for 2 nq queries, and with B200SA_APPROX_BEST 8
 * bytes per fetched entry for staging.  Phases: strand_queries after approx_check, strand_merge before end; the
 * other phases keep their names and meaning.
 *
 * ---- approximate document listing (DESIGN.md 6b f-19) ----
 * With B200SA_APPROX_DOCUMENTS (bit 29) in k, b200sa_docs_approx_positions_dev lists the documents that contain
 * each query within the threshold instead of the hits.  The flag is accepted by the documents entry alone, in any
 * mix with B200SA_APPROX_EDIT, B200SA_APPROX_BEST | B200SA_APPROX_SLACK(s), B200SA_APPROX_IUPAC and
 * B200SA_APPROX_BOTH_STRANDS; the threshold is decoded as without it.  On b200sa_approx_positions_dev bit 29 is an
 * unknown bit (B200SA_ERR_BAD_ARG, detail naming B200SA_APPROX_MAX_K); any other unknown bit on the documents
 * entry is B200SA_ERR_BAD_ARG with a detail that names B200SA_APPROX_MAX_K and B200SA_APPROX_DOCUMENTS.  Without
 * the flag nothing changes.  Definition:
 *  - L(q) is the list the same call with bit 29 cleared returns for q: entries (p, d(p)) by ascending p, or
 *    (p, d(p), strand) by (p, strand) with + first under B200SA_APPROX_BOTH_STRANDS.
 *  - doc(p) is the last d with doc_starts[d] <= p, as in b200sa_doc_ids_dev; an empty document holds no position
 *    and is never listed.
 *  - q's list has one entry per distinct doc(p) over L(q), by ascending document index: d_pos[i] is the document,
 *    d_mismatches[i] (may be NULL) the least d(p) over that document's entries of L(q), with B200SA_APPROX_MINUS
 *    set (under B200SA_APPROX_BOTH_STRANDS) exactly when no + entry of that document reaches that least distance:
 *    the document's first entry in (d, strand) order, + first.
 *  - With B200SA_APPROX_BEST, best(q) and t(q) are those of the call without the flag, over the whole collection,
 *    not per document: a document is listed iff it holds an occurrence at distance <= t(q).
 *  - Protocol: the listing protocol.  d_offsets (nq + 1, exclusive) and *total count documents and are always
 *    written; d_pos and d_mismatches are written only when total <= cap, never past total.  With cap = 0,
 *    offsets[q + 1] - offsets[q] is q's approximate document frequency.
 *  - Unchanged from the call without the flag: the other argument checks and error codes, the TOO_LARGE slot and
 *    query-length checks, nq = 0, n = 0, m = 0, the bytes read, synchronisation and the meaning of
 *    b200sa_last_stats().doubling_rounds.
 *  - So every document count is at most the call's hit count without the flag; at threshold 0 with the Hamming
 *    metric, one strand and no IUPAC, q's documents are those b200sa_docs_list_dev lists for q's exact range, each
 *    at distance 0; a palindromic query (rc(q) = q) never has B200SA_APPROX_MINUS set.
 * Method: q's final list is built as without the flag, but always emitted, into staging: ordered by p (or by
 * (p, strand)), so each document's hits are contiguous within a query.  One thread per staged hit marks the hits
 * that start a query's list or change document, a scan of the marks numbers the (query, document) segments and
 * gives the offsets, each segment start writes its document, and the least (d << 1) | minus of a segment is taken
 * with an atomicMin, so the result does not depend on the order of the hits.  Device workspace (computed, not
 * measured): what the fetch call without the flag takes for the whole hit list (even the cap = 0 call emits every
 * hit), plus 20 bytes per hit for the staged list, its marks and their scan, and 8 bytes per query.  Phases: those
 * of the call without the flag (with its emission phases even at cap = 0), then adocs_mark and, when the listing
 * fits, adocs_emit, before end.
 *
 * ---- alignments of the hits (DESIGN.md 6b f-20) ----
 * With B200SA_APPROX_ALIGN (bit 27) in k, b200sa_docs_approx_positions_dev lists the alignment operations of the
 * hits instead of the hits.  The flag is accepted by the documents entry alone, in any mix with
 * B200SA_APPROX_EDIT, B200SA_APPROX_BEST | B200SA_APPROX_SLACK(s), B200SA_APPROX_IUPAC and
 * B200SA_APPROX_BOTH_STRANDS; a single text goes through that entry as one document (doc_starts = {0}, ndocs = 1,
 * G = sa).  B200SA_APPROX_ALIGN | B200SA_APPROX_DOCUMENTS returns B200SA_ERR_BAD_ARG with a detail that names
 * both; on b200sa_approx_positions_dev bit 27 is an unknown bit as before.  Without the flag nothing changes.
 * Definition:
 *  - L(q) is the list the same call with bit 27 cleared returns for q: hits (p, d, strand) by p, or by
 *    (p, strand) with + first; best(q) and t(q) are that call's.
 *  - Q is q for a + hit and rc(q) for a - hit (the complement above, IUPAC classes included), m = |Q|, E = the
 *    end of p's document.  match(x, t) is T[t] == Q[x], or with B200SA_APPROX_IUPAC "T[t] is in the class of
 *    Q[x]" (only uppercase A C G T in the text match).
 *  - Hamming: window position x gives = if match(x, p + x), else X; end = p + m.
 *  - Edit: D(x, t) for 0 <= x <= m, p <= t <= E: D(m, t) = 0; D(x, E) = m - x; otherwise D(x, t) =
 *    min(D(x+1, t+1) + [not match(x, t)], D(x+1, t) + 1, D(x, t+1) + 1), so D(0, p) = d.  The canonical walk
 *    starts at (x, t) = (0, p) and, while x < m, takes the first move that holds: (1) t < E and D(x, t) =
 *    D(x+1, t+1) + [not match]: = or X, x+1, t+1; (2) D(x, t) = D(x+1, t) + 1: I (a query byte with no text
 *    byte), x+1; (3) otherwise D (a text byte with no query byte), t+1.  end = the final t.
 *  - Adjacent moves with one code merge into one operation.  Operations are in text order: a - hit's describe
 *    rc(q) against T[p, end), as SAM does for reverse-strand reads.  So the lengths of X, I and D sum to d, those of
 *    =, X and I to m, those of =, X and D to end - p; end <= E; the last operation is never D; a hit has at most
 *    2d + 1 operations (and at least one: m = 0 has no hits).
 *  - Band lemma: every cell the walk visits lies on a diagonal t - p - x in [-d, d] (each step off the diagonal
 *    costs 1).  A neighbour on an optimal continuation has an optimal path inside the band and one that is not
 *    fails the equality banded or not, so a DP over those 2d + 1 <= 63 diagonals, with values saturated at
 *    d + 1, takes the same walk.  The device recomputes D(0, p) and checks it against the staged d; a difference
 *    returns B200SA_ERR_INTERNAL, which is never expected.
 *  - Output, the listing protocol with operations as entries: d_offsets (nq + 1, exclusive) and *total count
 *    operations and are always written; entries go by hit as in L(q), and within a hit in walk order.  d_pos[i] is
 *    the hit's p, d_mismatches[i] the operation as a BAM word, len << 4 | code with I = 1, D = 2, = 7, X = 8,
 *    and B200SA_APPROX_MINUS on every operation of a - hit.  A hit is a maximal run of one query's entries with
 *    equal (p, minus).  d_pos and d_mismatches are written only when total <= cap, never past total;
 *    d_mismatches is required when cap > 0 (NULL returns B200SA_ERR_BAD_ARG).  cap = 0 counts only, but stages
 *    and aligns every hit, as B200SA_APPROX_DOCUMENTS does.
 *  - Limits, checked in phase approx_check: a query longer than 2^27 - 1 bytes (operation lengths leave bit 31
 *    for B200SA_APPROX_MINUS), or with B200SA_APPROX_EDIT longer than B200SA_APPROX_ALIGN_MAX_M bytes (the bound
 *    of the traceback's shared memory), returns B200SA_ERR_TOO_LARGE with a detail naming the limit.
 *  - Unchanged from the call without the flag: the other argument checks and error codes, nq = 0, n = 0, the
 *    bytes read, synchronisation and b200sa_last_stats().doubling_rounds.
 * Method: the final hit list is staged as with B200SA_APPROX_DOCUMENTS.  One count kernel aligns every hit and
 * keeps its merged words at a stride of 2 threshold + 1 words: Hamming one thread per hit; edit one warp per hit,
 * lane l holding diagonals l and l + 32, the row's deletion move a warp suffix-minimum scan, and each row's 2-bit
 * move choices (16 bytes) in shared memory, walked forward by one lane.  A scan of the counts gives each hit's
 * first entry and the offsets, and an emit kernel copies the words.  Device workspace (computed, not measured):
 * what the fetch call without the flag takes for the whole hit list, plus 20 bytes per hit for the staged list,
 * the counts and their scan, 4 (2 threshold + 1) bytes per hit for the words, and 8 bytes per query; with
 * B200SA_APPROX_EDIT, 16 bytes of shared memory per row of the longest query in the batch per resident warp
 * (64 KB per warp at B200SA_APPROX_ALIGN_MAX_M).  Phases: those of the call without the flag (with its emission
 * phases even at cap = 0), then align_count, align_scan and, when the listing fits, align_emit, before end.
 *
 * ---- fixed symbols in IUPAC queries (DESIGN.md 6b f-21) ----
 * With B200SA_APPROX_FIXED (bit 25) in k, b200sa_docs_approx_positions_dev keeps the lowercase symbols of each
 * query fixed: they must match their class, and the threshold is spent on the other symbols only.  This is the
 * usual definition of a CRISPR off-target (a PAM such as "ngg" must match; mismatches and bulges fall in the
 * spacer).  The flag is accepted by the documents entry alone, and only with B200SA_APPROX_IUPAC; alongside it
 * it mixes freely with B200SA_APPROX_EDIT, B200SA_APPROX_BEST | B200SA_APPROX_SLACK(s),
 * B200SA_APPROX_BOTH_STRANDS, B200SA_APPROX_DOCUMENTS and B200SA_APPROX_ALIGN.  A single text goes through that
 * entry as one document.  On b200sa_approx_positions_dev bit 25 is an unknown bit as before; without
 * B200SA_APPROX_IUPAC it returns B200SA_ERR_BAD_ARG with a detail that names both flags.  Without the flag nothing
 * changes.  Definition:
 *  - A query symbol is fixed when its byte is a lowercase IUPAC letter (a c g t u r y s w k m b d h v n), free
 *    when it is uppercase.  Classes do not change: lowercase means its uppercase class.  So a batch of uppercase
 *    queries means exactly what it means without the flag.
 *  - Hamming: p is an occurrence iff the window fits in its document, every fixed x has T[p + x] in the class of
 *    q[x], and mis(p), counted over the free x only, is at most the threshold.
 *  - Edit: dist(p) is the least cost of an alignment as above under three rules: a fixed symbol is aligned as =,
 *    never X or I; a text byte with no query byte (D) never sits directly before or after a fixed symbol (no D
 *    move at (x, t) when q[x] is fixed, or x >= 1 and q[x - 1] is fixed); when no alignment keeps the rules,
 *    dist(p) is infinite.
 *  - Everything else keeps its meaning on these distances: best(q) and t(q); the strands, rc(q) carrying its
 *    marks reversed (fixed(rc(q))[x] = fixed(q)[m - 1 - x]); the document listing; and the canonical walk of
 *    B200SA_APPROX_ALIGN, which takes its first allowed move.  So with B200SA_APPROX_ALIGN no X or I falls on a
 *    fixed position and no D touches one.
 *  - So a query with no lowercase symbol gives the call without the flag, bit for bit; the Hamming list is the
 *    list without the flag filtered to the windows whose fixed symbols match, at unchanged distances; and a query
 *    whose symbols are all fixed gives, under either metric at any threshold, the Hamming hits at threshold 0.
 * Method: a mark per query byte (1 = fixed), made from the original bytes beside the canonical copy, follows the
 * queries through the doubled batch of both strands (reversed for rc(q)), the compacted batches of the best
 * rounds and the alignment.  The pieces and reporters are those of B200SA_APPROX_IUPAC: the constrained
 * occurrences are a subset of the unconstrained ones, so one of the threshold + 1 pieces is still intact.
 * Verification rejects a window on a fixed miss and counts the free misses; the edit band DP and the alignment's
 * traceback forbid the three moves.  Device workspace (computed, not measured): what the call takes without the
 * flag, plus 1 byte per query byte for the marks (2 with B200SA_APPROX_BOTH_STRANDS, and as much again for a
 * compacted batch with B200SA_APPROX_BEST).  Phases: those of the call without the flag.
 *
 * ---- separate budgets for mismatches, DNA bulges and RNA bulges (DESIGN.md 6b f-22) ----
 * With B200SA_APPROX_BULGES (bit 21) | B200SA_APPROX_DNA_BULGES(d) | B200SA_APPROX_RNA_BULGES(r) in k, 0 <= d, r <= 3,
 * b200sa_docs_approx_positions_dev searches with three budgets, as CRISPR off-target tools do: the threshold t = k &
 * 0xFFFF counts substitutions alone, beside at most d DNA bulges and r RNA bulges.  The flag requires
 * B200SA_APPROX_EDIT and mixes freely with B200SA_APPROX_IUPAC, B200SA_APPROX_FIXED, B200SA_APPROX_BOTH_STRANDS,
 * B200SA_APPROX_DOCUMENTS and B200SA_APPROX_ALIGN; a single text goes through that entry as one document.  Each of
 * these returns B200SA_ERR_BAD_ARG with a detail that names B200SA_APPROX_BULGES: the flag without
 * B200SA_APPROX_EDIT; the flag with B200SA_APPROX_BEST (the detail names both); t + d + r > B200SA_APPROX_MAX_K; the
 * flag on b200sa_approx_positions_dev (an unknown bit there, whose detail also names B200SA_APPROX_MAX_K as before).
 * Bits 17-18 and 22-23 mean something only beside bit 21: without it they are unknown bits as before, with the same
 * detail.  Without the flag nothing changes.  Definition:
 *  - An alignment of the whole query Q (q, or rc(q) on a minus hit) to T[p, e), p <= e <= end(p), is made of =, X
 *    (a substitution), I (a query byte with no text byte: an RNA bulge) and D (a text byte with no query byte: a
 *    DNA bulge), with match as in B200SA_APPROX_ALIGN (IUPAC classes with B200SA_APPROX_IUPAC).
 *  - p is an occurrence when some alignment has #X <= t, #D <= d and #I <= r, and with B200SA_APPROX_FIXED also
 *    keeps the f-21 rules.  dist(p) is the least #X + #I + #D over those alignments; q's list holds (p, dist(p)) by
 *    ascending p, and both strands, the document listing and the listing protocol are as above on these
 *    distances.  m = 0 has no occurrences.
 *  - With B200SA_APPROX_ALIGN each hit gets the canonical alignment of cost dist(p) within the budgets: the walk
 *    from (0, p) takes, of the moves =/X, I, D in that order (f-20's), the first after which some alignment of the
 *    rest still keeps the remaining budgets at the remaining cost (with B200SA_APPROX_FIXED, the first allowed one).
 *    So every CIGAR has at most t X, d D and r I operations, and its X, I and D lengths sum to dist(p).
 *  - So: with d = r = 0 the call is exactly the Hamming call on the same entry with the same other flags,
 *    positions and distances bit for bit; the hits are a subset of the B200SA_APPROX_EDIT call at threshold
 *    t + d + r, each with dist(p) at least the edit distance there; the result only grows with t, d and r.
 *  - TOO_LARGE: the slot check counts nq * (t + d + r + 1) (2 nq with both strands).
 * Method: the pieces, slots and flow of B200SA_APPROX_EDIT with P = t + d + r + 1 pieces (the f-14 cut, or f-17's
 * with B200SA_APPROX_IUPAC; the whole-table slot when they do not fit).  A piece j found at s gives the starts p in
 * [c - d, c + r], c = s - o_j; the reporter rule is f-15's with the shift window s'' - o_i - p in [-r, d].  A banded
 * reversed Sellers DP over the 2(d + r) + 1 diagonals keeps, per cell and per (#I, #D) in [0..r] x [0..d], the least
 * #X, saturated at t + 1, in shared memory; the alignment recomputes the d + r + 1 diagonals of its hit, one thread
 * per hit, with every row kept in a device buffer of at most 64 MB per batch of hits.  Device workspace (computed,
 * not measured): what B200SA_APPROX_EDIT takes at threshold t + d + r, and with B200SA_APPROX_ALIGN up to 64 MB for
 * the rows.  Phases: those of the call without the flag.
 *
 * ---- one hit per locus (DESIGN.md 6b f-23) ----
 * With B200SA_APPROX_LOCI (bit 7) in k, b200sa_docs_approx_positions_dev lists one hit per locus instead of the run
 * of neighbouring starts that one site yields (an exact hit at p also puts p - 1 and p + 1 at distance 1 under
 * B200SA_APPROX_EDIT, and a bulge budget adds more), so that counts count sites.  On that entry the threshold is
 * k & 0xFF7F (k & 0x7F with B200SA_APPROX_BEST, and likewise the t of B200SA_APPROX_BULGES); on
 * b200sa_approx_positions_dev bit 7 stays a threshold bit, with its behaviour and error message unchanged.  The flag
 * mixes freely with B200SA_APPROX_EDIT, B200SA_APPROX_BEST | B200SA_APPROX_SLACK(s), B200SA_APPROX_IUPAC,
 * B200SA_APPROX_FIXED, B200SA_APPROX_BOTH_STRANDS, B200SA_APPROX_BULGES and B200SA_APPROX_ALIGN; a single text goes
 * through that entry as one document.  B200SA_APPROX_LOCI | B200SA_APPROX_DOCUMENTS returns B200SA_ERR_BAD_ARG with
 * a detail that names both (the document listing already keeps one entry per document).  Without the flag nothing
 * changes.  Definition:
 *  - L(q) is the list the same call with bit 7 cleared returns for q: hits (p, d, strand); best(q) and t(q) are
 *    that call's.  m = |q| in bytes.
 *  - Two hits of L(q) are linked when they are on the same strand, in the same document, and |p - p'| < m.  A locus
 *    is a maximal chain of linked hits: in ascending p, one strand's hits in one document, cut wherever consecutive
 *    starts differ by m or more.
 *  - Each locus is represented by its hit with the least d, ties going to the least p.  q's list is its
 *    representatives, ordered by (p, strand) with + first; each carries its own d, with B200SA_APPROX_MINUS on a
 *    - hit.
 *  - Protocol: the listing protocol; offsets and *total count loci.  With cap = 0 the call still stages every hit,
 *    as B200SA_APPROX_DOCUMENTS does.  With B200SA_APPROX_ALIGN the output is the representatives' alignments,
 *    exactly the words the call without bit 7 gives for those hits.
 *  - Unchanged from the call without the flag: the argument checks and error codes, the TOO_LARGE checks, nq = 0,
 *    n = 0, m = 0, the bytes read, synchronisation and b200sa_last_stats().doubling_rounds.
 *  - So the loci are a subset of L(q), at equal distances; if no two same-strand hits of q in one document are
 *    closer than m, the result is L(q) bit for bit; with m = 1 nothing merges; hits in different documents, or on
 *    different strands, never merge.
 * Method: the final list is staged as with B200SA_APPROX_DOCUMENTS.  Over the staged list, a max scan carries the
 * last hit index of each strand (one 32-bit channel per strand), which marks the heads: a hit whose previous hit of
 * its strand lies in another query or document, or m or more bytes before it.  A second max scan carries the last
 * head index of each strand, which gives each hit its locus, and the least (d << 32) | p of a locus is taken with an
 * atomicMin at its head, so the result does not depend on the order of the hits.  A chain as long as the text goes
 * through the scans' carries, never through a serial loop.  A sum scan of the representatives gives their places
 * and the offsets, and they are copied out (or, with B200SA_APPROX_ALIGN, back into staging for the alignment).
 * A call with 2^32 - 1 or more staged hits returns B200SA_ERR_TOO_LARGE.  Device workspace (computed, not measured):
 * what the call without the flag takes with the staged list (the fetch call's emission for the whole hit list, plus
 * the staging's 20 bytes per hit and 8 per query), plus 20 bytes per hit for the least keys, the scan of the
 * representatives and the heads, and with B200SA_APPROX_ALIGN 8 bytes per query.  Phases: those of the call without
 * the flag (with its emission phases even at cap = 0), then loci_mark and, when the listing fits or with
 * B200SA_APPROX_ALIGN, loci_emit, before the alignment's phases. */
#define B200SA_APPROX_MAX_K 31
#define B200SA_APPROX_EDIT 0x10000u
#define B200SA_APPROX_BEST 0x100000u                      /* bit 20 */
#define B200SA_APPROX_SLACK(s) ((uint32_t)(s) << 8)       /* 0 <= s <= 31, only with B200SA_APPROX_BEST */
#define B200SA_APPROX_IUPAC 0x1000000u                    /* bit 24 */
#define B200SA_APPROX_BOTH_STRANDS 0x10000000u            /* bit 28, in k */
#define B200SA_APPROX_MINUS 0x80000000u                   /* bit 31, in d_mismatches entries */
#define B200SA_APPROX_DOCUMENTS 0x20000000u               /* bit 29, in k, documents entry only */
#define B200SA_APPROX_ALIGN 0x8000000u                    /* bit 27, in k, documents entry only */
#define B200SA_APPROX_ALIGN_MAX_M 4096                    /* the longest query B200SA_APPROX_EDIT aligns */
#define B200SA_APPROX_FIXED 0x2000000u                    /* bit 25, in k, documents entry only, with B200SA_APPROX_IUPAC */
#define B200SA_APPROX_BULGES 0x200000u                    /* bit 21, in k, documents entry only, with B200SA_APPROX_EDIT */
#define B200SA_APPROX_DNA_BULGES(d) ((uint32_t)(d) << 17)  /* bits 17-18, 0 <= d <= 3, only with B200SA_APPROX_BULGES */
#define B200SA_APPROX_RNA_BULGES(r) ((uint32_t)(r) << 22)  /* bits 22-23, 0 <= r <= 3, only with B200SA_APPROX_BULGES */
#define B200SA_APPROX_LOCI 0x80u                          /* bit 7, in k, documents entry only */
int b200sa_approx_positions_dev(b200sa_ctx *ctx, const uint8_t *d_text, uint64_t n, const uint32_t *d_sa,
                                const uint8_t *d_queries, const uint64_t *d_q_off, uint32_t nq, uint32_t k,
                                uint64_t *d_offsets, uint32_t *d_pos, uint32_t *d_mismatches, uint64_t cap,
                                uint64_t *total, void *stream);
int b200sa_docs_approx_positions_dev(b200sa_ctx *ctx, const uint8_t *d_text, uint64_t n, const uint32_t *d_gsa,
                                     const uint32_t *d_doc_starts, uint32_t ndocs, const uint8_t *d_queries,
                                     const uint64_t *d_q_off, uint32_t nq, uint32_t k, uint64_t *d_offsets,
                                     uint32_t *d_pos, uint32_t *d_mismatches, uint64_t cap, uint64_t *total,
                                     void *stream);

/* ---- multi-GPU: communicator + sharded LMS-suffix sort (SURVEY.md 8e, config 5) ----
 * One process (or thread) and one context per GPU.  NCCL is resolved at run time
 * (the copy already loaded in the process, else libnccl.so.2); the single-GPU entry
 * points never touch it.  Either let the library create the communicator --
 * rank 0 calls b200sa_comm_unique_id, the application hands the 128 bytes to every
 * rank (MPI, torch.distributed, a file), every rank calls b200sa_comm_init -- or
 * attach an ncclComm_t the application already owns (same NCCL instance).
 *
 * b200sa_shard_lms_sort (collective): rank r passes its contiguous shard of the
 * text (rank order = text order; 16-byte aligned device pointer).  The shards are
 * classified (types, LMS positions; halo chars and carries exchanged), then the
 * LMS suffixes of the WHOLE text are ordered by their first kc characters (64-bit
 * window keys, zero-padded past the end of the text) with one sample-sort
 * exchange: rank r ends up with the r-th slice of the global order.
 *   d_sorted_gpos[i]  global text position of the i-th LMS suffix of this slice
 *   d_names[i]        dense global rank of its window (equal windows share a name)
 *   out->ties_total   members of groups of equal windows over all ranks; 0 means
 *                     the slices ARE the LMS suffixes in suffix order
 * Replaces, for a sharded text, src/table.rs:411-416 (LMS placement), :421-448
 * (first induce) and :450-482 (compaction + naming). */
typedef struct {
    uint64_t n_total;        /* bytes of the whole text                                 */
    uint64_t m_total;        /* LMS suffixes of the whole text                          */
    uint64_t m_local;        /* LMS suffixes of this shard                              */
    uint64_t lo;             /* global offset of this shard                             */
    uint64_t recv_count;     /* entries of this rank's slice of the global order        */
    uint64_t distinct_local; /* distinct windows in the slice                           */
    uint64_t name_offset;    /* distinct windows on lower ranks                         */
    uint64_t ties_total;     /* members of non-singleton window groups, all ranks       */
    double   bytes_sent;     /* payload this rank sent to OTHER ranks (NVLink)          */
    double   bytes_recv;
    uint32_t kc;             /* characters per window                                   */
    uint32_t nranks, rank;
    uint32_t reserved;
} b200sa_shard_stats;

int b200sa_comm_unique_id(uint8_t *id128_out);
int b200sa_comm_init(b200sa_ctx *ctx, int nranks, int rank, const uint8_t *id128);
int b200sa_comm_attach(b200sa_ctx *ctx, void *nccl_comm);
int b200sa_comm_destroy(b200sa_ctx *ctx);
int b200sa_shard_lms_sort(b200sa_ctx *ctx, const uint8_t *d_shard, uint64_t len,
                          unsigned long long *d_sorted_gpos, uint32_t *d_names, uint64_t cap,
                          b200sa_shard_stats *out, void *stream);

/* Sharded lcp_lens (collective; SURVEY.md 8e): d_text (n bytes), d_sa and d_lcp (n u32) are
 * device buffers on EVERY rank.  replicated == 0: rank 0 holds text and table, they are
 * broadcast first; != 0: every rank already holds them.  Every rank computes Phi / PLCP for
 * its own range of text positions, the ranges are all-gathered, every rank turns its range of
 * ranks into LCP values, the slices are all-gathered: on return every rank holds the whole
 * lcp array, equal to lcp_lens_quadratic(text, table) (src/table.rs:348-361). */
int b200sa_lcp_sharded(b200sa_ctx *ctx, uint8_t *d_text, uint64_t n, uint32_t *d_sa, uint32_t *d_lcp,
                       int replicated, void *stream);

/* ---- introspection (bench / tests) ---- */

typedef struct {
    uint64_t n;               /* text bytes of the last build                     */
    uint64_t m;               /* LMS suffixes at level 0                          */
    uint64_t names;           /* robust path: distinct LMS substrings (reduced alphabet);
                                 direct path: LMS suffixes settled by the first window */
    uint32_t doubling_rounds; /* robust path: rank-pair doubling rounds on the reduced
                                 string; direct path: window rounds of the LMS sort */
    uint32_t kernel_launches; /* kernels launched by the last call                */
    uint32_t induce_blocks;   /* grid of the persistent induce kernels            */
    uint32_t sm_count;
    uint64_t workspace_bytes; /* device workspace currently held                  */
    uint32_t direct_sort;     /* 1: LMS suffixes sorted directly by character windows;
                                 0: robust path (stage-1 induce + naming + doubling) */
    uint32_t reserved;
} b200sa_stats;

int b200sa_last_stats(b200sa_ctx *ctx, b200sa_stats *out);

/* Per-phase device times (CUDA events on the launching stream) of the last
 * call.  Enable with b200sa_set_timing(ctx, 1).  Returns the number of phases;
 * fills up to cap entries.  names[i] points to static strings. */
int b200sa_set_timing(b200sa_ctx *ctx, int enabled);
int b200sa_last_phase_times(b200sa_ctx *ctx, const char **names, float *ms, int cap);

const char *b200sa_strerror(int code);
const char *b200sa_last_error(b200sa_ctx *ctx);   /* detail of the last failure */
const char *b200sa_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200SA_H */
