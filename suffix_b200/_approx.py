"""Approximate positions (occurrences with at most k mismatches, or within k edits with metric="edit", with
best=s only each query's best hits, with iupac=True queries in IUPAC nucleotide codes, with fixed=True their
lowercase symbols fixed, with strands="both" the reverse complement's hits as well, and with loci=True one hit per
locus), the documents that hold them, and their alignments, over a device-resident table: the part SuffixTable and DocumentSuffixTable share.  A
table supplies `_device` and `_bwt_arrays()` -> (d_text, d_table, d_doc_starts or None, ndocs), its text and table
on the device; the LCP array is not needed."""
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
ALIGN = 0x8000000         # B200SA_APPROX_ALIGN
FIXED = 0x2000000         # B200SA_APPROX_FIXED
BULGES = 0x200000         # B200SA_APPROX_BULGES
LOCI = 0x80               # B200SA_APPROX_LOCI
MAX_BULGE = 3             # the most DNA or RNA bulges
OPS = "MIDNSHP=X"         # the BAM operation codes
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


def _fixed(fixed, iupac):
    """The k bit of fixed=: B200SA_APPROX_FIXED for True (which needs iupac=True), 0 for False."""
    if not isinstance(fixed, (bool, np.bool_)):
        raise ValueError("fixed must be True or False, got %r" % (fixed,))
    if fixed and not iupac:
        raise ValueError("fixed=True requires iupac=True")
    return FIXED if fixed else 0


def _bulges(bulges, k, metric, best):
    """The k bits of bulges=: 0 for None; for (dna, rna), two ints in 0 .. 3, B200SA_APPROX_BULGES with
    B200SA_APPROX_DNA_BULGES(dna) | B200SA_APPROX_RNA_BULGES(rna), which need metric="edit", best=None and
    k + dna + rna <= 31."""
    if bulges is None:
        return 0
    if (not isinstance(bulges, tuple) or len(bulges) != 2 or
            any(isinstance(b, (bool, np.bool_)) or not isinstance(b, (int, np.integer)) or not 0 <= b <= MAX_BULGE
                for b in bulges)):
        raise ValueError("bulges must be None or a tuple (dna, rna) of ints in 0 .. %d, got %r" % (MAX_BULGE, bulges))
    if metric != "edit":
        raise ValueError("bulges requires metric='edit'")
    if best is not None:
        raise ValueError("bulges does not combine with best")
    dna, rna = int(bulges[0]), int(bulges[1])
    if k + dna + rna > MAX_K:
        raise ValueError("k + dna + rna bulges must be at most %d, got %d" % (MAX_K, k + dna + rna))
    return BULGES | (dna << 17) | (rna << 22)


def _loci(loci):
    """The k bit of loci=: B200SA_APPROX_LOCI for True, 0 for False."""
    if not isinstance(loci, (bool, np.bool_)):
        raise ValueError("loci must be True or False, got %r" % (loci,))
    return LOCI if loci else 0


def _strands(strands):
    """The k bit of strands=: 0 for "forward", B200SA_APPROX_BOTH_STRANDS for "both"."""
    if not isinstance(strands, str) or strands not in ("forward", "both"):
        raise ValueError("strands must be 'forward' or 'both', got %r" % (strands,))
    return BOTH_STRANDS if strands == "both" else 0


def _call(table, queries, k, fetch, metric="hamming", best=None, iupac=False, strands="forward", documents=False,
          align=False, fixed=False, bulges=None, loci=False):
    """(offsets u64[nq + 1], positions u32[], distances u32[]); positions and distances are None without
    fetch (the cap = 0 call).  metric "hamming" counts mismatches, "edit" the Levenshtein distance; best=s keeps
    each query's occurrences within s of its least distance (include/b200sa.h, B200SA_APPROX_BEST); iupac=True reads
    the queries as IUPAC nucleotide codes, matched against the uppercase text bytes A C G T only
    (B200SA_APPROX_IUPAC); strands="both" adds the reverse complement's occurrences, the distances of those carrying
    B200SA_APPROX_MINUS (B200SA_APPROX_BOTH_STRANDS); documents=True (a DocumentSuffixTable only) lists the
    documents that hold q's hits instead, with the least distance in each (B200SA_APPROX_DOCUMENTS); align=True
    lists the alignment operations of q's hits instead, as (offsets, p, BAM word) entries (B200SA_APPROX_ALIGN);
    fixed=True (with iupac=True) keeps the lowercase query symbols fixed: they must match their class and take no
    edit, and the threshold is spent on the uppercase ones (B200SA_APPROX_FIXED); bulges=(dna, rna) (with
    metric="edit" and best=None) makes k the substitution budget beside at most dna DNA bulges (text bytes with no
    query byte) and rna RNA bulges (query bytes with no text byte) (B200SA_APPROX_BULGES); loci=True keeps one hit
    per locus, a chain of same-strand hits in one document whose starts are less than the query's length apart,
    the one with the least distance, leftmost on a tie (B200SA_APPROX_LOCI).  With align, fixed, bulges or loci a
    single text goes through the documents entry as one document."""
    import torch
    k = int(k)
    if not 0 <= k <= MAX_K:
        raise ValueError("k must be in 0 .. %d, got %d" % (MAX_K, k))
    if metric not in METRICS:
        raise ValueError("metric must be 'hamming' or 'edit', got %r" % (metric,))
    kf = (k | METRICS[metric] | _flags(best) | _iupac(iupac) | _fixed(fixed, iupac) | _strands(strands) |
          _bulges(bulges, k, metric, best) | _loci(loci) | (DOCUMENTS if documents else 0) | (ALIGN if align else 0))
    qs = [_as_bytes(q) for q in queries]
    nq, n = len(qs), len(table)
    d_t, d_r, d_s, ndocs = table._bwt_arrays()
    dev = torch.device("cuda", table._device)
    if (align or fixed or bulges is not None or loci) and d_s is None:
        d_s, ndocs = _one_document(table, dev), 1
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


def positions_batch(table, queries, k, metric="hamming", best=None, iupac=False, strands="forward", fixed=False,
                    bulges=None, loci=False):
    off, pos, dist = _call(table, queries, k, True, metric, best, iupac, strands, fixed=fixed, bulges=bulges,
                           loci=loci)
    if strands == "forward":
        return off, pos, dist
    return (off, pos) + _split(dist)


def positions(table, query, k, metric="hamming", best=None, iupac=False, strands="forward", fixed=False, bulges=None,
              loci=False):
    _, pos, dist = _call(table, [query], k, True, metric, best, iupac, strands, fixed=fixed, bulges=bulges, loci=loci)
    if strands == "forward":
        return pos, dist
    return (pos,) + _split(dist)


def counts(table, queries, k, metric="hamming", best=None, iupac=False, strands="forward", fixed=False, bulges=None,
           loci=False):
    off, _, _ = _call(table, queries, k, False, metric, best, iupac, strands, fixed=fixed, bulges=bulges, loci=loci)
    return np.diff(off.astype(np.int64)).astype(np.uint64)


def documents_batch(table, queries, k, metric="hamming", best=None, iupac=False, strands="forward", fixed=False):
    off, docs, dist = _call(table, queries, k, True, metric, best, iupac, strands, documents=True, fixed=fixed)
    if strands == "forward":
        return off, docs, dist
    return (off, docs) + _split(dist)


def documents(table, query, k, metric="hamming", best=None, iupac=False, strands="forward", fixed=False):
    _, docs, dist = _call(table, [query], k, True, metric, best, iupac, strands, documents=True, fixed=fixed)
    if strands == "forward":
        return docs, dist
    return (docs,) + _split(dist)


def document_frequencies(table, queries, k, metric="hamming", best=None, iupac=False, strands="forward", fixed=False):
    off, _, _ = _call(table, queries, k, False, metric, best, iupac, strands, documents=True, fixed=fixed)
    return np.diff(off.astype(np.int64)).astype(np.uint32)


def _one_document(table, dev):
    """doc_starts = {0} on the device, kept on the table: a single text as a collection of one document."""
    import torch
    if getattr(table, "_dev_one_doc", None) is None:
        table._dev_one_doc = torch.zeros(1, dtype=torch.int32, device=dev)
    return table._dev_one_doc


def cigar_string(words):
    """The CIGAR string of BAM words (len << 4 | code), e.g. "12=1X7=1I2="; bit 31 is ignored."""
    return "".join("%d%s" % ((int(w) & 0x7FFFFFFF) >> 4, OPS[int(w) & 15]) for w in words)


def _hits(off, pos, words):
    """The hits of an operation listing: (hit offsets u64[nq + 1], positions, distances, minus, ends,
    cigar_offsets u64[h + 1], cigar u32[]).  A hit is a maximal run of one query's entries with equal (p, minus);
    its distance is the length of its X, I and D operations, its end p plus that of =, X and D."""
    off = off.astype(np.int64)
    total = int(off[-1])
    q = np.repeat(np.arange(len(off) - 1), np.diff(off))
    minus = (words & np.uint32(MINUS)) != 0
    first = np.ones(total, dtype=bool)
    first[1:] = (q[1:] != q[:-1]) | (pos[1:] != pos[:-1]) | (minus[1:] != minus[:-1])
    starts = np.flatnonzero(first)
    hoff = np.concatenate([[0], np.cumsum(first)])[off].astype(np.uint64)
    cigar = words & np.uint32(MINUS - 1)
    lens, code = (cigar >> 4).astype(np.int64), cigar & np.uint32(15)
    if len(starts):
        dist = np.add.reduceat(np.where(code != 7, lens, 0), starts)
        span = np.add.reduceat(np.where(code != 1, lens, 0), starts)
    else:
        dist = span = np.zeros(0, dtype=np.int64)
    p = pos[starts]
    cigar_off = np.append(starts, total).astype(np.uint64)
    return (hoff, p, dist.astype(np.uint32), minus[starts], (p.astype(np.int64) + span).astype(np.uint32), cigar_off,
            cigar)


def alignments_batch(table, queries, k, metric="hamming", best=None, iupac=False, strands="forward", fixed=False):
    off, pos, words = _call(table, queries, k, True, metric, best, iupac, strands, align=True, fixed=fixed)
    hoff, p, dist, minus, ends, cigar_off, cigar = _hits(off, pos, words)
    if strands == "forward":
        return hoff, p, dist, ends, cigar_off, cigar
    return hoff, p, dist, minus, ends, cigar_off, cigar


def alignments(table, query, k, metric="hamming", best=None, iupac=False, strands="forward", fixed=False):
    return alignments_batch(table, [query], k, metric, best, iupac, strands, fixed)[1:]
