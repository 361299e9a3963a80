"""Generalized suffix array over many documents, without separators (SURVEY.md 8f-6).

The reference's README (README.md:60-74) names the generalized suffix array as missing and
offers a separator recipe instead (`GeneralizedSuffixTable`).  `DocumentSuffixTable` needs
no separator: documents may hold any bytes, a suffix ends at its document's end, equal
suffixes of different documents are ordered by document index, and the LCP array never
crosses a document end.  Construction (b200sa_docs_build) and batched queries
(b200sa_docs_positions_dev) run on the GPU; single queries run on the host like
`SuffixTable`'s.
"""
import bisect

import numpy as np

from . import _approx, _bwt, _lib, _lz, _match, _repeats
from .table import _as_bytes, _lock      # the lock of the per-device default context, shared with SuffixTable

MAX_N = 0xFFFFF000        # B200SA_MAX_N
TOPK_MAX = 1024           # B200SA_TOPK_MAX


class DocumentSuffixTable:
    """All positions of the concatenated documents, sorted by (document suffix, document)."""

    def __init__(self, docs, *, device: int = 0):
        docs = [_as_bytes(d) for d in docs]
        self._device = device
        self._text = b"".join(docs)
        if len(self._text) > MAX_N:
            raise OverflowError("documents longer than 2^32-4096 bytes in all (B200SA_MAX_N)")
        starts, pos = [], 0
        for d in docs:
            starts.append(pos)
            pos += len(d)
        self._starts = np.asarray(starts, dtype=np.uint32)
        self._ends = np.append(self._starts[1:], np.uint32(len(self._text))).astype(np.uint32) if docs else self._starts
        self._dev = None
        self._dev_lcp = None
        self._dlist = None
        t = np.frombuffer(self._text, dtype=np.uint8)
        with _lock:                           # default context is not thread-safe
            self._table, self._lcp = _lib.default_context(device).docs_build(t, self._starts, with_lcp=True)

    # ---- the table
    def table(self) -> np.ndarray:
        """G as u32 offsets into the concatenation of the documents."""
        return self._table

    def lcp_lens(self) -> np.ndarray:
        """lcp[0] = 0, lcp[i] = common prefix of the document suffixes G[i-1] and G[i]."""
        return self._lcp

    def text(self) -> bytes:
        """The concatenation of the documents."""
        return self._text

    def doc_starts(self) -> np.ndarray:
        return self._starts

    def __len__(self) -> int:
        return len(self._table)

    def len(self) -> int:
        return len(self._table)

    def is_empty(self) -> bool:
        return len(self._table) == 0

    def _doc_of(self, p: int) -> int:
        return bisect.bisect_right(self._starts, p) - 1     # the last document starting at or before p

    def _end_of(self, p: int) -> int:
        return int(self._ends[self._doc_of(p)])

    def suffix_bytes(self, i: int) -> bytes:
        """The suffix of entry i, cut at its document's end."""
        p = int(self._table[i])
        return self._text[p:self._end_of(p)]

    # ---- queries
    def _device_arrays(self):
        """Device copies of the concatenation, G and doc_starts, made on first use and kept while
        the table lives (so repeated batches do not copy them again)."""
        if self._dev is None:
            import torch
            dev = torch.device("cuda", self._device)
            up = lambda a: torch.from_numpy(a.copy()).to(dev)
            self._dev = (up(np.frombuffer(self._text or b"\0", dtype=np.uint8)), up(self._table.view(np.int32)),
                         up(self._starts.view(np.int32)))
        return self._dev

    def locate(self, positions) -> np.ndarray:
        """(document, offset) of each position of the concatenation (device batch)."""
        import torch
        p = np.ascontiguousarray(positions, dtype=np.uint32)
        if len(p) == 0 or len(self._starts) == 0:
            return np.zeros((0, 2), dtype=np.uint32)
        dev = torch.device("cuda", self._device)
        d_p = torch.from_numpy(p.view(np.int32).copy()).to(dev)
        d_s = self._device_arrays()[2]
        d_doc = torch.empty(len(p), dtype=torch.int32, device=dev)
        d_off = torch.empty(len(p), dtype=torch.int32, device=dev)
        with _lock:
            _lib.default_context(self._device).doc_ids_dev(d_p.data_ptr(), len(p), d_s.data_ptr(), len(self._starts),
                                                            d_doc.data_ptr(), d_off.data_ptr(),
                                                            torch.cuda.current_stream(dev).cuda_stream)
        torch.cuda.synchronize(dev)
        return np.stack([d_doc.cpu().numpy().view(np.uint32), d_off.cpu().numpy().view(np.uint32)], axis=1)

    def _head(self, i: int, m: int) -> bytes:
        p = int(self._table[i])
        return self._text[p:min(p + m, self._end_of(p))]

    def _range(self, q: bytes):
        """[start, end) of the entries whose document suffix starts with q (src/table.rs:223-259)."""
        n, m = len(self._table), len(q)
        if n == 0 or m == 0:
            return 0, 0
        h0 = self._head(0, m)
        if (q < h0 and not h0.startswith(q)) or q > self._head(n - 1, m):
            return 0, 0
        lo, hi = 0, n
        while lo < hi:                        # first entry >= q
            mid = (lo + hi) // 2
            if q <= self._head(mid, m):
                hi = mid
            else:
                lo = mid + 1
        start = lo
        lo, hi = 0, n - start
        while lo < hi:                        # first entry not starting with q
            mid = (lo + hi) // 2
            if self._head(start + mid, m) != q:
                hi = mid
            else:
                lo = mid + 1
        return start, start + lo

    def positions(self, query) -> np.ndarray:
        """(document, offset) rows of every occurrence of `query`, in table order."""
        s, e = self._range(_as_bytes(query))
        return self.locate(self._table[s:e])

    def contains(self, query) -> bool:
        return self.any_position(query) is not None

    def any_position(self, query):
        """(document, offset) of some occurrence of `query`, or None (src/table.rs:279-293)."""
        q = _as_bytes(query)
        m = len(q)
        if m == 0:
            return None
        lo, hi = 0, len(self._table)
        while lo < hi:
            mid = (lo + hi) // 2
            head = self._head(mid, m)
            if head == q:
                p = int(self._table[mid])
                d = self._doc_of(p)
                return d, p - int(self._starts[d])
            if head < q:
                lo = mid + 1
            else:
                hi = mid
        return None

    def positions_batch(self, queries):
        """Per query the range [start, end) of table() whose document suffixes start with it
        (b200sa_docs_positions_dev): two u32 arrays.  The first call copies the concatenation,
        G and doc_starts to the device; they stay there for later calls."""
        d_start, d_end = self._positions_dev(queries)
        return d_start.cpu().numpy().view(np.uint32), d_end.cpu().numpy().view(np.uint32)

    def _positions_dev(self, queries):
        """positions_batch with the ranges left on the device: two int32 tensors of u32 values."""
        import torch
        qs = [_as_bytes(q) for q in queries]
        nq = len(qs)
        dev = torch.device("cuda", self._device)
        if nq == 0:
            return torch.zeros(0, dtype=torch.int32, device=dev), torch.zeros(0, dtype=torch.int32, device=dev)
        off = np.zeros(nq + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(q) for q in qs])
        blob = np.frombuffer(b"".join(qs) or b"\0", dtype=np.uint8)
        n = len(self._text)
        d_t, d_g, d_s = self._device_arrays()
        d_q = torch.from_numpy(blob.copy()).to(dev)
        d_off = torch.from_numpy(off.view(np.int64)).to(dev)
        d_start = torch.empty(nq, dtype=torch.int32, device=dev)
        d_end = torch.empty(nq, dtype=torch.int32, device=dev)
        with _lock:
            _lib.default_context(self._device).docs_positions_dev(
                d_t.data_ptr(), n, d_g.data_ptr(), d_s.data_ptr(), len(self._starts), d_q.data_ptr(),
                d_off.data_ptr(), nq, d_start.data_ptr(), d_end.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        torch.cuda.synchronize(dev)
        return d_start, d_end

    # ---- document listing
    def _list_arrays(self):
        """byd and prev of b200sa_docs_list_index_dev (two int32 tensors of u32 values), built on the device
        on first use and kept while the table lives: 8 bytes per text byte of device memory."""
        if self._dlist is None:
            import torch
            d_t, d_g, d_s = self._device_arrays()
            dev = d_g.device
            n = len(self._table)
            byd = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
            prev = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
            with _lock:
                if self._dlist is None:
                    _lib.default_context(self._device).docs_list_index_dev(
                        n, d_g.data_ptr(), d_s.data_ptr(), len(self._starts), byd.data_ptr(), prev.data_ptr(),
                        torch.cuda.current_stream(dev).cuda_stream)
                    torch.cuda.synchronize(dev)
                    self._dlist = (byd, prev)
        return self._dlist

    def _list_dev(self, queries, cap_guess, with_tf=True):
        """_list_ranges_dev over the ranges of positions_batch."""
        d_start, d_end = self._positions_dev(queries)
        return self._list_ranges_dev(d_start, d_end, cap_guess, with_tf)

    def _list_ranges_dev(self, d_start, d_end, cap_guess, with_tf=True):
        """b200sa_docs_list_dev over ranges of table() on the device: (offsets, docs, tf) as device tensors
        (u64 offsets as int64, u32 entries as int32, tf None without with_tf).  cap_guess = 0 asks for the
        offsets alone; otherwise the buffers hold cap_guess entries and a larger listing is fetched by a
        second call sized to it."""
        import torch
        nq = len(d_start)
        dev = d_start.device
        d_off = torch.zeros(nq + 1, dtype=torch.int64, device=dev)
        if nq == 0:
            e = torch.zeros(0, dtype=torch.int32, device=dev)
            return d_off, e, e if with_tf else None
        byd, prev = self._list_arrays()
        _, d_g, d_s = self._device_arrays()
        n = len(self._table)

        def call(cap):
            docs = torch.empty(max(cap, 1), dtype=torch.int32, device=dev)
            tf = torch.empty(max(cap, 1), dtype=torch.int32, device=dev) if with_tf else None
            with _lock:
                total = _lib.default_context(self._device).docs_list_dev(
                    n, d_g.data_ptr(), d_s.data_ptr(), len(self._starts), byd.data_ptr(), prev.data_ptr(),
                    d_start.data_ptr(), d_end.data_ptr(), nq, d_off.data_ptr(), docs.data_ptr() if cap else 0,
                    tf.data_ptr() if cap and with_tf else 0, cap, torch.cuda.current_stream(dev).cuda_stream)
            return total, docs, tf

        total, docs, tf = call(cap_guess)
        if cap_guess and total > cap_guess:
            total, docs, tf = call(total)
        return d_off, docs[:total] if cap_guess else docs[:0], (tf[:total] if cap_guess else tf[:0]) if with_tf else None

    def documents_batch(self, queries, *, _cap_guess=None):
        """Per query the documents that contain it and its number of occurrences in each (overlapping
        occurrences count; a match never crosses a document end): (offsets u64[nq + 1], docs u32[],
        counts u32[]), query q's rows at [offsets[q], offsets[q+1]), sorted by document.  The listing runs
        on the device (b200sa_docs_list_dev, Muthukrishnan's array over the ranges of positions_batch); its
        index, built on the first call and kept, holds 8 bytes per text byte of device memory.  b"" lists
        nothing."""
        qs = list(queries)
        if _cap_guess is None:
            _cap_guess = max(1, min(1 << 24, 64 * len(qs)))
        return self._documents_sorted(*self._list_dev(qs, _cap_guess))

    def _ranges_dev(self, start, end):
        """Two equally long arrays of u32 range bounds as int32 device tensors."""
        import torch
        start = np.ascontiguousarray(start, dtype=np.uint32)
        end = np.ascontiguousarray(end, dtype=np.uint32)
        if start.shape != end.shape or start.ndim != 1:
            raise ValueError("start and end must be one-dimensional and equally long")
        dev = torch.device("cuda", self._device)
        return (torch.from_numpy(start.view(np.int32).copy()).to(dev),
                torch.from_numpy(end.view(np.int32).copy()).to(dev))

    def documents_for_ranges(self, start, end):
        """documents_batch for ranges [start[q], end[q]) of table() instead of query strings: the ranges that
        positions_batch, matching_statistics and smems return.  A range with start > end or end > len(self)
        is an error."""
        d_start, d_end = self._ranges_dev(start, end)
        return self._documents_sorted(*self._list_ranges_dev(d_start, d_end, max(1, min(1 << 24, 64 * len(d_start)))))

    def _documents_sorted(self, d_off, docs, tf):
        """The listing of _list_ranges_dev by ascending document per query, on the host."""
        import torch
        nq = len(d_off) - 1
        if len(docs):
            # rank order -> document order per query: one sort of (query, document) keys
            q = torch.repeat_interleave(torch.arange(nq, device=docs.device, dtype=torch.int64), d_off.diff())
            key = (q << 32) | (docs.to(torch.int64) & 0xFFFFFFFF)
            order = torch.argsort(key)
            docs, tf = docs[order], tf[order]
        torch.cuda.synchronize(docs.device)
        return (d_off.cpu().numpy().view(np.uint64), docs.cpu().numpy().view(np.uint32),
                tf.cpu().numpy().view(np.uint32))

    def documents(self, query) -> np.ndarray:
        """(document, count) rows of the documents that contain `query`, by ascending document: a batch of one."""
        _, docs, tf = self.documents_batch([query])
        return np.stack([docs, tf], axis=1)

    def document_frequencies(self, queries) -> np.ndarray:
        """For each query, the number of documents that contain it (0 for b""): the listing's counts alone
        (b200sa_docs_list_dev with cap = 0), without building the tree of DocumentSuffixTree."""
        d_off, _, _ = self._list_dev(list(queries), 0, with_tf=False)
        return d_off.diff().cpu().numpy().astype(np.uint32)

    # ---- top-k document retrieval
    def top_documents_batch(self, queries, k):
        """Per query the min(k, df) documents that contain it most often, by occurrence count descending and
        then by ascending document: (offsets u64[nq + 1], docs u32[], counts u32[]), query q's rows at
        [offsets[q], offsets[q+1]) in that order.  1 <= k <= TOPK_MAX (for a longer answer use
        documents_batch).  Runs on the device (b200sa_docs_topk_dev over the ranges of positions_batch) with
        the index of documents_batch; the device output is nq * k rows, whatever the listing's size.  b"" and
        absent queries have no rows."""
        import torch
        k = int(k)
        if not 1 <= k <= TOPK_MAX:
            raise ValueError("k must be in 1 .. %d, got %d" % (TOPK_MAX, k))
        return self._top_ranges_dev(*self._positions_dev(queries), k)

    def top_documents_for_ranges(self, start, end, k):
        """top_documents_batch for ranges [start[q], end[q]) of table() instead of query strings (see
        documents_for_ranges)."""
        k = int(k)
        if not 1 <= k <= TOPK_MAX:
            raise ValueError("k must be in 1 .. %d, got %d" % (TOPK_MAX, k))
        return self._top_ranges_dev(*self._ranges_dev(start, end), k)

    def _top_ranges_dev(self, d_start, d_end, k):
        """b200sa_docs_topk_dev over ranges of table() on the device, compacted to the host triple."""
        import torch
        nq = len(d_start)
        if nq == 0:
            return np.zeros(1, dtype=np.uint64), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint32)
        dev = d_start.device
        byd, prev = self._list_arrays()
        _, d_g, d_s = self._device_arrays()
        count = torch.empty(nq, dtype=torch.int32, device=dev)
        docs = torch.empty(nq * k, dtype=torch.int32, device=dev)
        tf = torch.empty(nq * k, dtype=torch.int32, device=dev)
        with _lock:
            _lib.default_context(self._device).docs_topk_dev(
                len(self._table), d_g.data_ptr(), d_s.data_ptr(), len(self._starts), byd.data_ptr(), prev.data_ptr(),
                d_start.data_ptr(), d_end.data_ptr(), nq, k, count.data_ptr(), docs.data_ptr(), tf.data_ptr(),
                torch.cuda.current_stream(dev).cuda_stream)
        keep = torch.arange(k, device=dev, dtype=torch.int32)[None, :] < count[:, None]
        off = torch.zeros(nq + 1, dtype=torch.int64, device=dev)
        off[1:] = torch.cumsum(count, 0)
        docs, tf = docs.view(nq, k)[keep], tf.view(nq, k)[keep]
        torch.cuda.synchronize(dev)
        return off.cpu().numpy().view(np.uint64), docs.cpu().numpy().view(np.uint32), tf.cpu().numpy().view(np.uint32)

    # ---- matching statistics and SMEMs (DESIGN 6b f-10)
    def _match_call(self, ctx, d_q, d_off, nq, q_bytes, d_len, d_start, d_end, stream):
        import torch
        d_t, d_g, d_s = self._device_arrays()
        if self._dev_lcp is None:                 # glcp joins the device copies on first use: 4 bytes per text byte
            self._dev_lcp = torch.from_numpy(self._lcp.view(np.int32).copy()).to(d_g.device)
        ctx.docs_match_stats_dev(d_t.data_ptr(), len(self._table), d_g.data_ptr(), self._dev_lcp.data_ptr(),
                                 d_s.data_ptr(), len(self._starts), d_q, d_off, nq, q_bytes, d_len, d_start, d_end,
                                 stream)

    def matching_statistics(self, queries):
        """For every byte of every query, the longest piece starting there that occurs inside one document,
        and where (b200sa_docs_match_stats_dev): (offsets u64[nq + 1], length u32[], start u32[], end u32[]),
        the row of query q, offset j at offsets[q] + j.  table()[start:end] are the occurrences of
        query[j:j + length], the range positions_batch returns for that string ((0, 0) when length = 0)."""
        self._device_arrays()
        return _match.matching_statistics(self, queries)

    def smems(self, queries, min_len=1):
        """The super-maximal exact matches of every query: its matches of at least min_len bytes that lie
        inside no other match of the same query (b200sa_smems_dev).  (offsets u64[nq + 1], qpos u32[],
        length u32[], start u32[], end u32[]): query q's rows are [offsets[q], offsets[q+1]) by ascending
        qpos.  start / end feed documents_for_ranges and top_documents_for_ranges as they are."""
        self._device_arrays()
        return _match.smems(self, queries, min_len)

    # ---- repeats (DESIGN 6b f-11)
    _REPEAT_MODES = ("any", "earlier", "other_document", "earlier_document")

    def _repeat_arrays(self):
        import torch
        _, d_g, d_s = self._device_arrays()
        if self._dev_lcp is None:                 # glcp joins the device copies on first use: 4 bytes per text byte
            self._dev_lcp = torch.from_numpy(self._lcp.view(np.int32).copy()).to(d_g.device)
        return d_g, self._dev_lcp, d_s, len(self._starts)

    def repeat_lengths(self) -> np.ndarray:
        """u32[n]: for every position p of the concatenation, the longest prefix of p's document suffix
        that also starts at another position, in any document (b200sa_repeat_lens_dev)."""
        return _repeats.repeat_lengths(self)

    def repeated_substrings(self, min_len, with_ends=False):
        """The distinct strings of min_len bytes that occur at least twice inside documents, as ranges of
        the table (b200sa_repeat_runs_dev): (start u32[], end u32[]) in ascending order, or (start, end,
        first, last) with the smallest and largest position of each.  The ranges feed documents_for_ranges
        and top_documents_for_ranges as they are."""
        return _repeats.repeated_substrings(self, min_len, with_ends)

    def duplicate_spans(self, min_len, mode="any") -> np.ndarray:
        """(document, begin_offset, end_offset) rows, by document and offset: the maximal spans of bytes
        covered by a flagged position's next min_len bytes; a span never crosses a document end
        (b200sa_duplicate_spans_dev).  mode: "any" flags every position whose next min_len bytes occur at
        another position, "earlier" every such occurrence but the first, "other_document" those that
        occur in a different document, "earlier_document" those that occur in a document of smaller index."""
        begin, end = _repeats.duplicate_spans(self, min_len, mode, self._REPEAT_MODES)
        at = self.locate(begin)
        return np.concatenate([at, (at[:, 1] + (end - begin))[:, None]], axis=1).astype(np.uint32)

    def duplicated_bytes(self, min_len, mode="any") -> int:
        """The number of bytes duplicate_spans(min_len, mode) covers, without fetching the spans."""
        return _repeats.duplicated_bytes(self, min_len, mode, self._REPEAT_MODES)

    # ---- longest previous factor and LZ77 (DESIGN 6b f-12)
    def longest_previous_factors(self):
        """(lpf u32[n], src u32[n]) over the concatenation: lpf[p] is the longest prefix of p's document
        suffix that also starts at some q < p, in p's document or an earlier one (the occurrence may
        overlap p); src[p] is one such q, 0xFFFFFFFF where lpf[p] = 0 (b200sa_lpf_dev).  No factor
        crosses a document end."""
        return _lz.longest_previous_factors(self)

    def lz77_factors(self, *, _cap_guess=None):
        """(start u32[z], length u32[z], source u32[z]): the LZ77 factorization of the collection, with
        sources in any earlier position (b200sa_lz77_dev).  Positions are in coordinates of the
        concatenation, locate() maps them to (document, offset); every non-empty document starts a factor
        and no factor crosses a document end.  A literal has length 1 and source 0xFFFFFFFF."""
        return _lz.lz77_factors(self, _cap_guess)

    def lz77_count(self) -> int:
        """z, the number of LZ77 factors, without fetching them."""
        return _lz.lz77_count(self)

    # ---- Burrows-Wheeler transform (DESIGN 6b f-13)
    def _bwt_arrays(self):
        d_t, d_g, d_s = self._device_arrays()
        return d_t, d_g, d_s, len(self._starts)

    def bwt(self):
        """(bwt bytes[n], term_rows u32[k]): the multi-string Burrows-Wheeler transform of the documents, each
        ended by a terminator of its own, $_0 < $_1 < ... < every byte (b200sa_bwt_dev).  The rows are the k
        terminator rows followed by table()'s order; bwt holds the n bytes of L with the terminators left
        out, term_rows[d] the row whose L is $_d.  suffix_b200.inverse_bwt_documents(bwt, term_rows) gives
        the documents back."""
        return _bwt.bwt(self)

    def bwt_runs(self) -> int:
        """r, the number of maximal runs of equal symbols in the transform's n + k symbols; every terminator
        is a symbol of its own."""
        return _bwt.bwt_runs(self)

    # ---- approximate positions (DESIGN 6b f-14 .. f-21)
    def approximate_positions(self, query, k, *, metric="hamming", best=None, iupac=False, strands="forward",
                              fixed=False, bulges=None, loci=False):
        """(positions u32[], mismatches u32[]): every position p of the concatenation whose window of m bytes
        lies inside p's document and differs from the query (m bytes) in at most k bytes, 0 <= k <= 31, by
        ascending p, with that number of mismatches beside it (b200sa_docs_approx_positions_dev).  locate()
        maps the positions to (document, offset).  b"" matches nothing.  metric="edit": every p with
        dist(p) <= k instead, dist(p) the least Levenshtein distance between the query and a substring that
        starts at p and ends inside p's document, listed beside p.  Any other metric than "hamming" or "edit"
        raises ValueError.
        best=s (an int, 0 <= s <= 31) lists only each query's best hits: with best(q) its least distance within
        k, the occurrences at distance <= min(k, best(q) + s), exactly what the call returns at that threshold
        (B200SA_APPROX_BEST).  best=0 gives each query's best hits, and the distance column then holds best(q)
        on every one.  best=None (the default) lists every occurrence within k; any other value, True included,
        raises ValueError.
        iupac=True reads each query byte as an IUPAC nucleotide code (A C G T, U = T, R Y S W K M B D H V N, in
        either case), which matches the uppercase text bytes A C G T of its class (B200SA_APPROX_IUPAC); any
        other query byte raises B200SA_ERR_BAD_ARG.  Lowercase (soft-masked) text bases, N, U and every other
        text byte match no code and count as a mismatch: uppercase a soft-masked text before building the
        table.  Combines with metric= and best=; a non-bool value raises ValueError.
        fixed=True (with iupac=True; a non-bool value, or fixed=True without iupac=True, raises ValueError) keeps
        the lowercase symbols of each query fixed (B200SA_APPROX_FIXED, the text going through
        b200sa_docs_approx_positions_dev as one document on a SuffixTable): a lowercase code still means its
        uppercase class, but must match it, and takes no substitution, insertion or adjacent deletion, so the
        threshold is spent on the uppercase symbols alone.  A CRISPR guide written "GACGCTGACGCTGACGCTGAngg"
        finds off-targets whose PAM is intact, with mismatches and bulges in the spacer only.  A query with no
        lowercase symbol gives exactly the call without the flag.
        bulges=(dna, rna) (two ints in 0 .. 3; needs metric="edit", best=None and k + dna + rna <= 31; any
        other value than None raises ValueError) searches as CRISPR off-target tools do, with three budgets in
        place of one (B200SA_APPROX_BULGES, the text going through b200sa_docs_approx_positions_dev as one
        document on a SuffixTable): p is listed when some alignment of the query to a text[p:e] has at most k
        substitutions, at most dna DNA bulges (text bases with no query base) and at most rna RNA bulges (query
        bases with no text base), with the least total of the three over those alignments beside it.
        bulges=(0, 0) gives exactly the Hamming call; combines with iupac=, fixed= and strands=.
        loci=True (a non-bool value raises ValueError) lists one hit per locus in place of the run of
        neighbouring starts that one site yields (B200SA_APPROX_LOCI): a locus is a
        chain of hits on one strand in one document whose consecutive starts are less than the query's length
        apart, and its hit with the least distance, the leftmost on a tie, represents it.  So a planted site gives
        one hit under metric="edit" and bulges= as under Hamming, and approximate_counts counts sites.  The result
        is a subset of the call without it, at equal distances; combines with every other keyword.
        strands="both" also lists the occurrences of the query's reverse complement (A <-> T, C <-> G in either
        case; with iupac=True each code's class complemented, R <-> Y, K <-> M, B <-> V, D <-> H, U -> A) as
        minus-strand hits at the leftmost text position of their window or alignment
        (B200SA_APPROX_BOTH_STRANDS), and returns (positions, distances, minus): one list by (p, strand) with
        the plus hit first, minus a bool array; with best= best(q) is taken over both strands.  strands="forward"
        (the default) searches the query alone; any other value raises ValueError."""
        return _approx.positions(self, query, k, metric, best, iupac, strands, fixed, bulges, loci)

    def approximate_positions_batch(self, queries, k, *, metric="hamming", best=None, iupac=False, strands="forward",
                                    fixed=False, bulges=None, loci=False):
        """(offsets u64[nq + 1], positions u32[], mismatches u32[]): query q's occurrences with at most k
        mismatches (or within k edits, metric="edit") are positions[offsets[q]:offsets[q + 1]], as
        approximate_positions returns them; best=0 gives each query's best hits, with best(q) in the
        distance column (best=, iupac=, fixed=, bulges= and loci= as in approximate_positions).  strands="both" returns (offsets,
        positions, distances, minus) with both strands in each query's list, as approximate_positions does."""
        return _approx.positions_batch(self, queries, k, metric, best, iupac, strands, fixed, bulges, loci)

    def approximate_counts(self, queries, k, *, metric="hamming", best=None, iupac=False, strands="forward",
                           fixed=False, bulges=None, loci=False):
        """u64[nq]: the number of occurrences with at most k mismatches (or within k edits, metric="edit") of
        every query, without fetching them; best=0 counts each query's best hits, those at distance best(q)
        (best=, iupac=, fixed= and bulges= as in approximate_positions); strands="both" counts the hits of both strands;
        loci=True counts loci, the sites that approximate_positions(loci=True) lists."""
        return _approx.counts(self, queries, k, metric, best, iupac, strands, fixed, bulges, loci)

    def approximate_alignments(self, query, k, *, metric="hamming", best=None, iupac=False, strands="forward"):
        """(positions u32[], distances u32[], ends u32[], cigar_offsets u64[h + 1], cigar u32[]): the hits of
        approximate_positions, in its order, each with its alignment (B200SA_APPROX_ALIGN, computed on the
        device).  Hit i aligns the query to text[positions[i]:ends[i]]; its operations are
        cigar[cigar_offsets[i]:cigar_offsets[i + 1]], BAM words len << 4 | code (I 1, D 2, = 7, X 8), in text
        order; suffix_b200.cigar_string turns them into "12=1X7=".  With metric="edit" the alignment is the
        canonical walk of include/b200sa.h, which prefers a substitution or match, then an insertion, then a
        deletion; the query must then be at most 4096 bytes (B200SA_APPROX_ALIGN_MAX_M).  distances and ends are
        read off the operations.  strands="both" returns (positions, distances, minus, ends, cigar_offsets,
        cigar), and a minus hit's operations align the reverse complement, as SAM does.  Keywords are checked as
        in approximate_positions."""
        return _approx.alignments(self, query, k, metric, best, iupac, strands)

    def approximate_alignments_batch(self, queries, k, *, metric="hamming", best=None, iupac=False,
                                     strands="forward"):
        """(offsets u64[nq + 1], positions, distances, ends, cigar_offsets, cigar): query q's hits are
        [offsets[q], offsets[q + 1]) of positions, distances and ends, as approximate_alignments returns them;
        one count call, then one fetch call sized by it.  strands="both" puts minus after distances."""
        return _approx.alignments_batch(self, queries, k, metric, best, iupac, strands)

    def approximate_documents(self, query, k, *, metric="hamming", best=None, iupac=False, strands="forward"):
        """(documents u32[], distances u32[]): the documents that hold an occurrence of the query within k, as
        approximate_positions finds them, by ascending document, each with the least distance of its
        occurrences there (b200sa_docs_approx_positions_dev with B200SA_APPROX_DOCUMENTS).  The listing is
        made on the device from the hits, which never cross PCIe.  Empty documents are never listed.  With
        best=s, best(q) and its threshold are those of approximate_positions, taken over the whole collection:
        a document is listed iff it holds a hit at distance <= min(k, best(q) + s).  strands="both" returns
        (documents, distances, minus), minus set when the least distance in that document is reached on the
        minus strand only.  metric=, best=, iupac= and strands= are checked as in approximate_positions."""
        return _approx.documents(self, query, k, metric, best, iupac, strands)

    def approximate_documents_batch(self, queries, k, *, metric="hamming", best=None, iupac=False,
                                    strands="forward"):
        """(offsets u64[nq + 1], documents u32[], distances u32[]): query q's documents are
        documents[offsets[q]:offsets[q + 1]], as approximate_documents returns them; one count call, then one
        fetch call sized by it.  strands="both" returns (offsets, documents, distances, minus)."""
        return _approx.documents_batch(self, queries, k, metric, best, iupac, strands)

    def approximate_document_frequencies(self, queries, k, *, metric="hamming", best=None, iupac=False,
                                         strands="forward"):
        """u32[nq]: the number of documents that hold an occurrence of each query within k (keywords as in
        approximate_documents), from the count call alone, without fetching the listing."""
        return _approx.document_frequencies(self, queries, k, metric, best, iupac, strands)

    def top_documents(self, query, k) -> np.ndarray:
        """(document, count) rows of the min(k, df) documents that contain `query` most often, by count
        descending, then by ascending document: a batch of one."""
        _, docs, tf = self.top_documents_batch([query], k)
        return np.stack([docs, tf], axis=1)

    def __repr__(self):
        return "DocumentSuffixTable(docs=%d, n=%d)" % (len(self._starts), len(self._table))
