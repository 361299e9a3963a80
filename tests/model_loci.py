"""Host statement of one hit per locus (include/b200sa.h, B200SA_APPROX_LOCI): collapse() applies the definition
to a packed listing (offsets, pos, d | MINUS on a minus hit) of any model or serial C statement -- hits linked when
on one strand, in one document and less than m = |q| apart, each maximal chain represented by its hit with the
least d, the leftmost on a tie -- in numpy, so that it runs over millions of hits.  keep_ops() filters an alignment
listing (B200SA_APPROX_ALIGN) to the hits that collapse() keeps."""
import numpy as np

MINUS = 0x80000000                      # B200SA_APPROX_MINUS


def _hit_queries(off):
    off = np.asarray(off, dtype=np.int64)
    return np.repeat(np.arange(len(off) - 1, dtype=np.int64), np.diff(off))


def keep_mask(packed, lengths, starts):
    """bool[total]: the representatives of the listing packed (offsets, pos, d | MINUS), queries of byte lengths
    lengths, documents starting at starts (None or empty: one document)."""
    off, pos, dist = packed
    pos = np.asarray(pos, dtype=np.int64)
    dist = np.asarray(dist, dtype=np.uint32)
    total = len(pos)
    if total == 0:
        return np.zeros(0, dtype=bool)
    q = _hit_queries(off)
    minus = (dist >> 31).astype(np.int64)
    d = (dist & np.uint32(MINUS - 1)).astype(np.int64)
    starts = np.zeros(1, np.int64) if starts is None or len(starts) == 0 else np.asarray(starts, dtype=np.int64)
    doc = np.searchsorted(starts, pos, side="right") - 1
    m = np.asarray(lengths, dtype=np.int64)[q]
    order = np.lexsort((pos, minus, q))                      # by (query, strand, p): each chain is contiguous
    qs, ss, ps, ds, ms = q[order], minus[order], pos[order], doc[order], m[order]
    head = np.ones(total, dtype=bool)
    head[1:] = (qs[1:] != qs[:-1]) | (ss[1:] != ss[:-1]) | (ds[1:] != ds[:-1]) | (ps[1:] - ps[:-1] >= ms[1:])
    locus = np.cumsum(head) - 1
    best = np.lexsort((ps, d[order], locus))                 # by (locus, d, p): the first of each locus wins
    first = np.ones(total, dtype=bool)
    first[1:] = locus[best][1:] != locus[best][:-1]
    keep = np.zeros(total, dtype=bool)
    keep[order[best[first]]] = True
    return keep


def collapse(packed, queries, starts=None):
    """The listing of the call with B200SA_APPROX_LOCI from that of the same call without it: packed (offsets, pos,
    d | MINUS), queries the query bytes (or their lengths), starts the document starts (None: one text)."""
    off, pos, dist = packed
    lengths = [q if isinstance(q, (int, np.integer)) else len(q) for q in queries]
    keep = keep_mask(packed, lengths, starts)
    q = _hit_queries(off)
    new_off = np.zeros(len(off), dtype=np.uint64)
    new_off[1:] = np.cumsum(np.bincount(q[keep], minlength=len(off) - 1))
    return new_off, np.asarray(pos, dtype=np.uint32)[keep], np.asarray(dist, dtype=np.uint32)[keep]


def keep_ops(ops, kept):
    """The alignment listing ops (offsets, p, BAM word | MINUS per operation, as B200SA_APPROX_ALIGN gives it)
    filtered to the hits (query, p, strand) of the listing kept."""
    off, pos, words = ops
    koff, kpos, kdist = kept
    kq = _hit_queries(koff)
    want = set(zip(kq.tolist(), np.asarray(kpos).tolist(), (np.asarray(kdist, np.uint32) >> 31).tolist()))
    q = _hit_queries(off)
    words = np.asarray(words, dtype=np.uint32)
    mask = np.array([h in want for h in zip(q.tolist(), np.asarray(pos).tolist(), (words >> 31).tolist())], dtype=bool)
    new_off = np.zeros(len(off), dtype=np.uint64)
    new_off[1:] = np.cumsum(np.bincount(q[mask], minlength=len(off) - 1))
    return new_off, np.asarray(pos, dtype=np.uint32)[mask], words[mask]
