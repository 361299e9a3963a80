"""Host statements of the approximate document listing (include/b200sa.h, B200SA_APPROX_DOCUMENTS): (a) the
definition applied to the list L(q) of the call without the flag -- one entry per distinct doc(p) over L(q), by
ascending document, with the least distance there and B200SA_APPROX_MINUS exactly when no plus entry of that
document reaches it -- composed from tests/model_strand.py and tests/model_best.py, (b) the same rule vectorised
over a whole packed result, for large sets, and (c) the device's rule: marks, their exclusive scan and a segment
minimum of (d << 1) | minus."""
import numpy as np

from tests import model_approx, model_best, model_strand

MINUS = model_strand.MINUS


def starts_of(docs):
    """doc_starts of the concatenation of docs."""
    return np.cumsum([0] + [len(d) for d in docs[:-1]]).astype(np.int64) if docs else np.zeros(0, np.int64)


def doc_of(starts, p):
    """The last d with starts[d] <= p."""
    return int(np.searchsorted(starts, p, side="right")) - 1


def flagless(docs, queries, k, metric="hamming", iupac=False, best=None, strands="forward"):
    """L(q) of every query, packed (offsets, pos, d | MINUS on a minus hit): the call with bit 29 cleared."""
    if strands == "both":
        return model_strand.brute(docs, queries, k, metric, iupac, best)
    packed = model_strand.one_strand(docs, queries, k, metric, iupac)
    if best is None:
        return packed
    out = []
    for h in model_best.lists(packed):
        t = model_best.threshold(min(d for _, d in h), k, best) if h else -1
        out.append([(p, d) for p, d in h if d <= t])
    return model_approx._pack(out)


def reduce_lists(packed, starts):
    """The definition, per query: [(document, least d | MINUS when only a minus entry reaches it)]."""
    out = []
    for h in model_best.lists(packed):
        per = {}
        for p, d in h:
            doc = doc_of(starts, p)
            key = ((d & (MINUS - 1)) << 1) | (d >> 31)
            per[doc] = min(per.get(doc, key), key)
        out.append([(doc, (w >> 1) | (MINUS if w & 1 else 0)) for doc, w in sorted(per.items())])
    return out


def brute(docs, queries, k, metric="hamming", iupac=False, best=None, strands="forward"):
    """(offsets, documents, distances) of the call with B200SA_APPROX_DOCUMENTS."""
    return model_approx._pack(reduce_lists(flagless(docs, queries, k, metric, iupac, best, strands), starts_of(docs)))


def group(packed, starts):
    """reduce_lists over a whole packed result at once (numpy), for large sets: (offsets, documents, distances)."""
    off, pos, dist = packed
    off = np.asarray(off, dtype=np.int64)
    pos = np.asarray(pos, dtype=np.int64)
    dist = np.asarray(dist, dtype=np.uint32)
    nq = len(off) - 1
    q = np.repeat(np.arange(nq), np.diff(off))
    d = np.searchsorted(np.asarray(starts, dtype=np.int64), pos, side="right") - 1
    key = ((dist & np.uint32(MINUS - 1)).astype(np.int64) << 1) | (dist >> 31).astype(np.int64)
    order = np.lexsort((key, d, q))
    q, d, key = q[order], d[order], key[order]
    first = np.ones(len(q), dtype=bool)
    first[1:] = (q[1:] != q[:-1]) | (d[1:] != d[:-1])
    q, d, key = q[first], d[first], key[first]
    out_off = np.zeros(nq + 1, dtype=np.uint64)
    out_off[1:] = np.cumsum(np.bincount(q, minlength=nq))
    dist_out = (key >> 1).astype(np.uint32) | np.where(key & 1, np.uint32(MINUS), np.uint32(0))
    return out_off, d.astype(np.uint32), dist_out


def device_rule(packed, starts):
    """The kernels' rule: mark[i] = hit i starts its query's list or changes document; seg = the exclusive scan of
    the marks; offsets[q] = seg[off[q]]; hit i is in segment seg[i + 1] - 1, whose document its start writes and
    whose word is the least (d << 1) | minus of its hits."""
    off, pos, dist = packed
    off = np.asarray(off, dtype=np.int64)
    nq, total = len(off) - 1, int(off[-1])
    q_of = np.repeat(np.arange(nq), np.diff(off))
    doc = [doc_of(starts, int(p)) for p in pos]
    mark = [1 if i == off[q_of[i]] or doc[i] != doc[i - 1] else 0 for i in range(total)]
    seg = np.zeros(total + 1, dtype=np.int64)
    seg[1:] = np.cumsum(mark)
    nseg = int(seg[-1])
    docs_out, least = [None] * nseg, [0xFFFFFFFF] * nseg
    for i in range(total):
        if seg[i + 1] != seg[i]:
            docs_out[seg[i]] = doc[i]
        d = int(dist[i])
        least[seg[i + 1] - 1] = min(least[seg[i + 1] - 1], ((d & (MINUS - 1)) << 1) | (d >> 31))
    dist_out = [(w >> 1) | (MINUS if w & 1 else 0) for w in least]
    return (seg[off].astype(np.uint64), np.asarray(docs_out, dtype=np.uint32),
            np.asarray(dist_out, dtype=np.uint32))
