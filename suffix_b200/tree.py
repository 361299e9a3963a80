"""Host-side mirror of the reference's `suffix_tree` crate (suffix_tree/src/lib.rs).

The tree is built on the GPU from the suffix table and its LCP array
(b200sa_suffix_tree, rules 1-8 in include/b200sa.h) and kept as six u32 arrays
indexed by preorder id; `Node` is a light (tree, id) handle over them.  The
reference's behaviours that are not textbook are kept:

- the root has an empty label and the terminal [n] (suffix_tree :84);
- there is no terminator character, so a suffix that is a proper prefix of the
  next one in SA order stays a terminal of a node that has children
  (:128-131, :432);
- `leaves()` skips the root because it only yields nodes with len() > 0 (:357).
"""
import numpy as np

from . import _lib
from .table import SuffixTable, _lock

NONE = 0xFFFFFFFF


class SuffixTree:
    """A suffix tree (suffix_tree/src/lib.rs:46-49)."""

    def __init__(self, text, *, device: int = 0):
        """SuffixTree::new (:67-72) == from_suffix_table(SuffixTable::new(text))."""
        self._init(SuffixTable(text, device=device))

    @classmethod
    def from_suffix_table(cls, table: SuffixTable) -> "SuffixTree":
        """SuffixTree::from_suffix_table (:74-76): built from table() and lcp_lens()."""
        st = cls.__new__(cls)
        st._init(table)
        return st

    def _init(self, table: SuffixTable):
        self._text = table.text()
        self._table = np.asarray(table.table(), dtype=np.uint32)
        lcp = table.lcp_lens()
        with _lock:
            a = _lib.default_context(table._device).suffix_tree(self._table, lcp)
        self._parent = a["parent"]
        self._depth = a["depth"]
        self._sa_lo = a["sa_lo"]
        self._sa_hi = a["sa_hi"]
        self._label_start = a["label_start"]
        self._subtree_end = a["subtree_end"]

    # ---- tree methods (:87-100)
    def text(self) -> bytes:
        return self._text

    def root(self) -> "Node":
        return self._node(self, 0)

    def label(self, node: "Node") -> bytes:
        """The path label into `node` (:97-100)."""
        s = int(self._label_start[node.id])
        return self._text[s:s + node.len()]

    def __len__(self) -> int:
        """Number of nodes, the root included."""
        return len(self._parent)

    def arrays(self) -> dict:
        """The six arrays by preorder id: parent, depth, sa_lo, sa_hi, label_start, subtree_end."""
        return {"parent": self._parent, "depth": self._depth, "sa_lo": self._sa_lo, "sa_hi": self._sa_hi,
                "label_start": self._label_start, "subtree_end": self._subtree_end}

    def __repr__(self) -> str:
        """The reference's Debug output of SuffixTree (:230-255); labels print as Rust's Debug of &[u8]."""
        out = ["\n-----------------------------------------\n", "SUFFIX TREE\n",
               "text: %s\n" % self._text.decode("utf-8", errors="replace"), "ROOT\n"]
        ends = []                                   # subtree ends of the open ancestors
        for v in range(1, len(self._parent)):
            while ends and ends[-1] <= v:
                ends.pop()
            ends.append(int(self._subtree_end[v]))
            lab = self.label(Node(self, v))
            out.append("  " * len(ends) + "[" + ", ".join(str(b) for b in lab) + "]\n")
        out.append("-----------------------------------------\n")
        return "".join(out)


class Node:
    """A node of a SuffixTree (:52-59): the tree and a preorder id."""

    __slots__ = ("tree", "id")

    def __init__(self, tree: SuffixTree, id: int):
        self.tree = tree
        self.id = int(id)

    def __eq__(self, other):
        return isinstance(other, Node) and other.tree is self.tree and other.id == self.id

    def __hash__(self):
        return hash((id(self.tree), self.id))

    def __repr__(self):
        return "Node(id=%d)" % self.id

    def parent(self):
        p = int(self.tree._parent[self.id])
        return None if p == NONE else type(self)(self.tree, p)

    def children(self):
        """Children in byte order of their labels' first bytes (:108-111)."""
        t = self.tree
        end = int(t._subtree_end[self.id])
        c = self.id + 1
        while c < end:
            yield type(self)(t, c)
            c = int(t._subtree_end[c])

    def ancestors(self):
        """This node, its parent, ..., the root (:113-118)."""
        t, v = self.tree, self.id
        while v != NONE:
            yield type(self)(t, v)
            v = int(t._parent[v])

    def preorder(self):
        """This node and its descendants in preorder, which is lexicographic (:120-125)."""
        t = self.tree
        for v in range(self.id, int(t._subtree_end[self.id])):
            yield type(self)(t, v)

    def leaves(self):
        """Nodes of the preorder with len() > 0 and terminals; they may have children (:127-134, :357)."""
        return (v for v in self.preorder() if v.len() > 0 and v.has_terminals())

    def suffix_indices(self) -> np.ndarray:
        """All suffix indices below this node, in the order of the reference's leaf walk (:136-139)."""
        t = self.tree
        return t._table[int(t._sa_lo[self.id]):int(t._sa_hi[self.id])]

    def len(self) -> int:
        """Length of the path label into this node (:141-144)."""
        t = self.tree
        p = int(t._parent[self.id])
        return 0 if p == NONE else int(t._depth[self.id]) - int(t._depth[p])

    def depth(self) -> int:
        """Number of ancestors, not counting this node (:146-149)."""
        return sum(1 for _ in self.ancestors()) - 1

    def has_terminals(self) -> bool:
        return len(self.suffixes()) > 0

    def suffixes(self) -> list:
        """Terminal suffix indices (:156-159): [n] at the root, else [sa[sa_lo]] or []."""
        t = self.tree
        n = len(t._table)
        if self.id == 0:
            return [n]
        s = int(t._table[int(t._sa_lo[self.id])])
        return [s] if int(t._depth[self.id]) == n - s else []


SuffixTree._node = Node          # the handle class of a tree's nodes (DocumentSuffixTree uses its own)
