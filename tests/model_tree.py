"""Pure-Python statement of rules 1-8 of include/b200sa.h: the reference's suffix tree
(suffix_tree/src/lib.rs:392-505) from SA + LCP, with stack-based ANSV so that it runs in
O(n).  It is the specification the CUDA kernels (suffix_b200/csrc/tree.cuh) implement."""
import numpy as np

NONE = 0xFFFFFFFF
FIELDS = ("parent", "depth", "sa_lo", "sa_hi", "label_start", "subtree_end")


def _ansv(L, n):
    psv, pse, nsv = [NONE] * n, [NONE] * n, [n] * n
    st = []
    for i in range(n):                       # strict: largest j < i with L[j] < L[i]
        while st and L[st[-1]] >= L[i]:
            st.pop()
        psv[i] = st[-1] if st else NONE
        st.append(i)
    st = []
    for i in range(n):                       # non-strict: largest j < i with L[j] <= L[i]
        while st and L[st[-1]] > L[i]:
            st.pop()
        pse[i] = st[-1] if st else NONE
        st.append(i)
    st = []
    for i in range(n - 1, -1, -1):           # strict: smallest j > i with L[j] < L[i]
        while st and L[st[-1]] >= L[i]:
            st.pop()
        nsv[i] = st[-1] if st else n
        st.append(i)
    return psv, pse, nsv


def tree_arrays(sa, lcp) -> dict:
    sa = [int(x) for x in sa]
    n = len(sa)
    if n == 0:
        return {f: np.array([v], dtype=np.uint32) for f, v in zip(FIELDS, (NONE, 0, 0, 0, 0, 1))}
    L = [int(x) for x in lcp] + [0]          # lcp[n] := 0
    psv, pse, nsv = _ansv(L, n)
    # rules 1-3: (depth, hi) of the nodes by sa_lo
    by_lo = [[] for _ in range(n)]
    by_lo[0].append((0, n))                  # root
    for i in range(1, n):
        if L[i] > 0 and pse[i] == psv[i]:
            by_lo[psv[i]].append((L[i], nsv[i]))
    for r in range(n):
        if not (r + 1 < n and L[r + 1] == n - sa[r]):
            by_lo[r].append((n - sa[r], r + 1))
    # rule 4: preorder = ascending (sa_lo, depth); a chain of nested nodes per sa_lo
    lo_of, dep, hi_of, first, ident = [], [], [], [0] * (n + 1), {}
    for lo in range(n):
        first[lo] = len(lo_of)
        for d, hi in sorted(by_lo[lo]):
            ident[(lo, d)] = len(lo_of)
            lo_of.append(lo)
            dep.append(d)
            hi_of.append(hi)
    N = len(lo_of)
    first[n] = N
    parent, label_start, subtree_end = [NONE] * N, [0] * N, [N] * N
    for v in range(1, N):
        lo, hi, d = lo_of[v], hi_of[v], dep[v]
        pd = max(L[lo], L[hi])               # rule 5
        if pd == 0:
            parent[v] = 0
        else:
            plo = lo if L[hi] > L[lo] else psv[lo]
            parent[v] = ident[(plo, pd)]
        label_start[v] = sa[lo] + pd         # rule 6
        subtree_end[v] = first[hi] if hi < n else N   # rule 7
    return {f: np.array(a, dtype=np.uint32)
            for f, a in zip(FIELDS, (parent, dep, lo_of, hi_of, label_start, subtree_end))}


def children(a: dict, v: int):
    """Rule 8."""
    c, end, se = v + 1, int(a["subtree_end"][v]), a["subtree_end"]
    while c < end:
        yield c
        c = int(se[c])
