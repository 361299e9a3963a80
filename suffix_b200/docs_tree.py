"""Generalized suffix tree of many documents, with the number of documents below every node
(SURVEY.md 8f-7).

`DocumentSuffixTree` is the compressed trie of the document suffixes of a `DocumentSuffixTable`:
suffixes end at their document's end, and equal suffixes of different documents share one node,
whose terminals are all of them.  It keeps the reference's no-terminator convention (a suffix that
is a proper prefix of another stays a terminal of a node with children; `suffixes()` is a list) and
its `SuffixTree` / `Node` API.  Each node also knows how many distinct documents lie below it, which
answers document frequency (`document_counts`, batched on the device) and the longest string shared
by at least k documents (`longest_common_substring`).  The tree and the counts are built on the GPU
(b200sa_docs_tree, rules in include/b200sa.h).
"""
import numpy as np

from . import _lib
from .docs import DocumentSuffixTable
from .table import _lock      # the lock of the per-device default context, shared with SuffixTable
from .tree import Node, SuffixTree


class DocumentNode(Node):
    """A node of a DocumentSuffixTree: terminals are G[sa_lo, term_end), possibly several documents'."""

    __slots__ = ()

    def has_terminals(self) -> bool:
        t = self.tree
        return int(t._term_end[self.id]) > int(t._sa_lo[self.id])

    def suffixes(self) -> list:
        """Terminal positions (offsets into the concatenation), in document order; [] at the root."""
        t = self.tree
        return t._table[int(t._sa_lo[self.id]):int(t._term_end[self.id])].tolist()

    def terminals(self) -> np.ndarray:
        """(document, offset) rows of the terminals."""
        t = self.tree
        return t._dst.locate(t._table[int(t._sa_lo[self.id]):int(t._term_end[self.id])])

    def doc_count(self) -> int:
        """Number of distinct documents among suffix_indices()."""
        return int(self.tree._doc_count[self.id])


class DocumentSuffixTree(SuffixTree):
    """The generalized suffix tree of a list of documents (any bytes, possibly empty)."""

    _node = DocumentNode

    def __init__(self, docs, *, device: int = 0):
        self._init_docs(DocumentSuffixTable(docs, device=device))

    @classmethod
    def from_document_table(cls, dst: DocumentSuffixTable) -> "DocumentSuffixTree":
        """The tree of a DocumentSuffixTable's table() and lcp_lens()."""
        st = cls.__new__(cls)
        st._init_docs(dst)
        return st

    def _init_docs(self, dst: DocumentSuffixTable):
        self._dst = dst
        self._text = dst.text()
        self._table = np.asarray(dst.table(), dtype=np.uint32)
        with _lock:
            a = _lib.default_context(dst._device).docs_tree(self._table, dst.lcp_lens(), dst.doc_starts())
        self._parent = a["parent"]
        self._depth = a["depth"]
        self._sa_lo = a["sa_lo"]
        self._sa_hi = a["sa_hi"]
        self._label_start = a["label_start"]
        self._subtree_end = a["subtree_end"]
        self._term_end = a["term_end"]
        self._doc_count = a["doc_count"]
        self._dev = None

    def document_table(self) -> DocumentSuffixTable:
        return self._dst

    def arrays(self) -> dict:
        """The eight arrays by preorder id: the six of SuffixTree, term_end and doc_count."""
        a = super().arrays()
        a["term_end"] = self._term_end
        a["doc_count"] = self._doc_count
        return a

    def _device_arrays(self):
        """Device copies of sa_lo, sa_hi and doc_count, made on first use and kept while the tree lives."""
        if self._dev is None:
            import torch
            dev = torch.device("cuda", self._dst._device)
            up = lambda a: torch.from_numpy(a.view(np.int32).copy()).to(dev)
            self._dev = (up(self._sa_lo), up(self._sa_hi), up(self._doc_count))
        return self._dev

    def document_counts(self, queries) -> np.ndarray:
        """For each query, the number of documents that contain it (0 for b""): the range search of
        DocumentSuffixTable.positions_batch and the node lookup both run on the device."""
        import torch
        d_start, d_end = self._dst._positions_dev(queries)
        nq = len(d_start)
        if nq == 0:
            return np.zeros(0, dtype=np.uint32)
        dev = d_start.device
        d_lo, d_hi, d_cnt = self._device_arrays()
        d_out = torch.empty(nq, dtype=torch.int32, device=dev)
        with _lock:
            _lib.default_context(self._dst._device).docs_tree_counts_dev(
                d_lo.data_ptr(), d_hi.data_ptr(), d_cnt.data_ptr(), len(self._sa_lo), d_start.data_ptr(),
                d_end.data_ptr(), nq, d_out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        torch.cuda.synchronize(dev)
        return d_out.cpu().numpy().view(np.uint32)

    def longest_common_substring(self, k: int) -> bytes:
        """The string of the deepest node below which at least k documents lie (the lowest preorder
        id among equally deep ones): a longest string that occurs in at least k documents.  b"" if
        no non-empty string does."""
        ok = np.nonzero(self._doc_count >= k)[0]
        if len(ok) == 0:
            return b""
        v = int(ok[np.argmax(self._depth[ok])])
        d = int(self._depth[v])
        if d == 0:
            return b""
        s = int(self._table[int(self._sa_lo[v])])
        return self._text[s:s + d]
