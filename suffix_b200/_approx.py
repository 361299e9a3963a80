"""Approximate positions (occurrences with at most k mismatches, or within k edits with metric="edit", with
best=s only each query's best hits, with iupac=True queries in IUPAC nucleotide codes, and with strands="both" the
reverse complement's hits as well), and the documents that hold them, over a device-resident
table: the part SuffixTable and DocumentSuffixTable share.  A table supplies `_device` and
`_bwt_arrays()` -> (d_text, d_table, d_doc_starts or None, ndocs), its text and table on the device; the LCP
array is not needed."""
import numpy as np

from . import _lib
from .table import _as_bytes, _lock

MAX_K = 31                # B200SA_APPROX_MAX_K
EDIT = 0x10000            # B200SA_APPROX_EDIT
BEST = 0x100000           # B200SA_APPROX_BEST
IUPAC = 0x1000000         # B200SA_APPROX_IUPAC
BOTH_STRANDS = 0x10000000  # B200SA_APPROX_BOTH_STRANDS
MINUS = 0x80000000        # B200SA_APPROX_MINUS
DOCUMENTS = 0x20000000    # B200SA_APPROX_DOCUMENTS
METRICS = {"hamming": 0, "edit": EDIT}


def _flags(best):
    """The k bits of best=: 0 for None, B200SA_APPROX_SLACK(s) | B200SA_APPROX_BEST for an int s in 0 .. 31."""
    if best is None:
        return 0
    if isinstance(best, (bool, np.bool_)) or not isinstance(best, (int, np.integer)) or not 0 <= best <= MAX_K:
        raise ValueError("best must be None or an int slack in 0 .. %d, got %r" % (MAX_K, best))
    return (int(best) << 8) | BEST


def _iupac(iupac):
    """The k bit of iupac=: B200SA_APPROX_IUPAC for True, 0 for False."""
    if not isinstance(iupac, (bool, np.bool_)):
        raise ValueError("iupac must be True or False, got %r" % (iupac,))
    return IUPAC if iupac else 0


def _strands(strands):
    """The k bit of strands=: 0 for "forward", B200SA_APPROX_BOTH_STRANDS for "both"."""
    if not isinstance(strands, str) or strands not in ("forward", "both"):
        raise ValueError("strands must be 'forward' or 'both', got %r" % (strands,))
    return BOTH_STRANDS if strands == "both" else 0


def _call(table, queries, k, fetch, metric="hamming", best=None, iupac=False, strands="forward", documents=False):
    """(offsets u64[nq + 1], positions u32[], distances u32[]); positions and distances are None without
    fetch (the cap = 0 call).  metric "hamming" counts mismatches, "edit" the Levenshtein distance; best=s keeps
    each query's occurrences within s of its least distance (include/b200sa.h, B200SA_APPROX_BEST); iupac=True reads
    the queries as IUPAC nucleotide codes, matched against the uppercase text bytes A C G T only
    (B200SA_APPROX_IUPAC); strands="both" adds the reverse complement's occurrences, the distances of those carrying
    B200SA_APPROX_MINUS (B200SA_APPROX_BOTH_STRANDS); documents=True (a DocumentSuffixTable only) lists the
    documents that hold q's hits instead, with the least distance in each (B200SA_APPROX_DOCUMENTS)."""
    import torch
    k = int(k)
    if not 0 <= k <= MAX_K:
        raise ValueError("k must be in 0 .. %d, got %d" % (MAX_K, k))
    if metric not in METRICS:
        raise ValueError("metric must be 'hamming' or 'edit', got %r" % (metric,))
    kf = k | METRICS[metric] | _flags(best) | _iupac(iupac) | _strands(strands) | (DOCUMENTS if documents else 0)
    qs = [_as_bytes(q) for q in queries]
    nq, n = len(qs), len(table)
    d_t, d_r, d_s, ndocs = table._bwt_arrays()
    dev = torch.device("cuda", table._device)
    off = np.zeros(nq + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(q) for q in qs])
    d_q = torch.from_numpy(np.frombuffer(b"".join(qs) or b"\0", dtype=np.uint8).copy()).to(dev)
    d_off = torch.from_numpy(off.view(np.int64)).to(dev)
    d_o = torch.zeros(nq + 1, dtype=torch.int64, device=dev)
    ctx = _lib.default_context(table._device)
    stream = torch.cuda.current_stream(dev).cuda_stream

    def call(cap, d_pos=0, d_mis=0):
        if d_s is None:
            return ctx.approx_positions_dev(d_t.data_ptr(), n, d_r.data_ptr(), d_q.data_ptr(), d_off.data_ptr(), nq,
                                            kf, d_o.data_ptr(), d_pos, d_mis, cap, stream)
        return ctx.docs_approx_positions_dev(d_t.data_ptr(), n, d_r.data_ptr(), d_s.data_ptr(), ndocs,
                                             d_q.data_ptr(), d_off.data_ptr(), nq, kf, d_o.data_ptr(), d_pos, d_mis,
                                             cap, stream)

    pos = mis = None
    with _lock:                                   # count, then fetch into buffers of that size
        total = call(0)
        if fetch:
            pos = torch.empty(max(total, 1), dtype=torch.int32, device=dev)
            mis = torch.empty(max(total, 1), dtype=torch.int32, device=dev)
            if total:
                call(total, pos.data_ptr(), mis.data_ptr())
    torch.cuda.synchronize(dev)
    offsets = d_o.cpu().numpy().view(np.uint64)
    if not fetch:
        return offsets, None, None
    return offsets, pos[:total].cpu().numpy().view(np.uint32), mis[:total].cpu().numpy().view(np.uint32)


def _split(dist):
    """(distances with B200SA_APPROX_MINUS cleared, minus bool[])"""
    return dist & np.uint32(MINUS - 1), (dist & np.uint32(MINUS)) != 0


def positions_batch(table, queries, k, metric="hamming", best=None, iupac=False, strands="forward"):
    off, pos, dist = _call(table, queries, k, True, metric, best, iupac, strands)
    if strands == "forward":
        return off, pos, dist
    return (off, pos) + _split(dist)


def positions(table, query, k, metric="hamming", best=None, iupac=False, strands="forward"):
    _, pos, dist = _call(table, [query], k, True, metric, best, iupac, strands)
    if strands == "forward":
        return pos, dist
    return (pos,) + _split(dist)


def counts(table, queries, k, metric="hamming", best=None, iupac=False, strands="forward"):
    off, _, _ = _call(table, queries, k, False, metric, best, iupac, strands)
    return np.diff(off.astype(np.int64)).astype(np.uint64)


def documents_batch(table, queries, k, metric="hamming", best=None, iupac=False, strands="forward"):
    off, docs, dist = _call(table, queries, k, True, metric, best, iupac, strands, documents=True)
    if strands == "forward":
        return off, docs, dist
    return (off, docs) + _split(dist)


def documents(table, query, k, metric="hamming", best=None, iupac=False, strands="forward"):
    _, docs, dist = _call(table, [query], k, True, metric, best, iupac, strands, documents=True)
    if strands == "forward":
        return docs, dist
    return (docs,) + _split(dist)


def document_frequencies(table, queries, k, metric="hamming", best=None, iupac=False, strands="forward"):
    off, _, _ = _call(table, queries, k, False, metric, best, iupac, strands, documents=True)
    return np.diff(off.astype(np.int64)).astype(np.uint32)
