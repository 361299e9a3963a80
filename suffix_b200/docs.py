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

from . import _lib
from .table import _as_bytes, _lock      # the lock of the per-device default context, shared with SuffixTable

MAX_N = 0xFFFFF000        # B200SA_MAX_N


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
        import torch
        qs = [_as_bytes(q) for q in queries]
        nq = len(qs)
        if nq == 0:
            return np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint32)
        off = np.zeros(nq + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(q) for q in qs])
        blob = np.frombuffer(b"".join(qs) or b"\0", dtype=np.uint8)
        dev = torch.device("cuda", self._device)
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
        return d_start.cpu().numpy().view(np.uint32), d_end.cpu().numpy().view(np.uint32)

    def __repr__(self):
        return "DocumentSuffixTable(docs=%d, n=%d)" % (len(self._starts), len(self._table))
