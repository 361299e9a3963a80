/*
 * b200sa_internal.h -- test / diagnostic hooks exported by libb200sa.so.
 * Not part of the drop-in boundary (that is b200sa.h); used by tests/ to
 * check each device primitive against numpy / the oracle in isolation.
 * All pointers are HOST buffers; every hook runs the CUDA kernels (there is
 * no CPU path) and copies results back.
 */
#ifndef B200SA_INTERNAL_H
#define B200SA_INTERNAL_H

#include <stdint.h>
#include "b200sa.h"

#ifdef __cplusplus
extern "C" {
#endif

/* K1/K2: classification of `text` by the fused single-pass byte classifier (classify2.cuh;
 * reference SuffixTypes::compute, src/table.rs:592-615; Bins::find_sizes, :686-704).
 * stype_words/lms_words: ceil(n/32) u32 bitmaps; hist768: L / S-non-LMS / LMS counts per byte;
 * lmspos_desc: up to cap_lms LMS positions in DESCENDING text order (the order the LMS sort is
 * fed in); *m_out their number. */
int b200sa_test_classify_fused(b200sa_ctx *ctx, const uint8_t *text, uint64_t n,
                               uint32_t *stype_words, uint32_t *lms_words, uint32_t *hist768,
                               uint32_t *lmspos_desc, uint64_t cap_lms, uint64_t *m_out);

/* Generic scan: op 0 = exclusive sum, op 1 = exclusive max; *total = reduction. */
int b200sa_test_scan(b200sa_ctx *ctx, const uint32_t *in, uint64_t n, int op,
                     uint32_t *out_excl, uint32_t *total);

/* Stable LSD radix sort of (key,value) pairs on the low `bits` key bits. */
int b200sa_test_sort_pairs32(b200sa_ctx *ctx, uint32_t *keys, uint32_t *vals, uint64_t n, int bits);
int b200sa_test_sort_pairs64(b200sa_ctx *ctx, uint64_t *keys, uint32_t *vals, uint64_t n, int bits);

/* Suffix array of a u32 string by rank-pair doubling (the reduced-problem
 * solver).  names = alphabet bound (all R[i] < names). */
int b200sa_test_reduced_sa(b200sa_ctx *ctx, const uint32_t *R, uint64_t m, uint32_t names,
                           uint32_t *sa_out, uint32_t *rounds_out);

/* Copies an internal device array of the last build to `out` (cap elements of
 * the array's element type); returns the element count or a negative error.
 * which: 0 lmspos(u32)  1 sorted LMS substrings(u32)  2 reduced string(u32)
 *        3 reduced SA(u32)  4 sorted LMS suffixes(u32)  5 induce err[4](u32)
 *        6 bucket tables bstart[257]|Lcnt[256]|Scnt[256]|lms_off[257](u32) */
int64_t b200sa_debug_fetch(b200sa_ctx *ctx, int which, void *out, uint64_t cap);

#ifdef __cplusplus
}
#endif
#endif /* B200SA_INTERNAL_H */
