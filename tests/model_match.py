"""Host statements of matching statistics and SMEMs (include/b200sa.h, b200sa_match_stats_dev /
b200sa_docs_match_stats_dev / b200sa_smems_dev): the definition by brute force, and a pure-Python model of
the device steps (suffix_b200/csrc/match.cuh) on (G, glcp) from model_docs.brute.  A single text is the
document set [text]."""
import numpy as np

from tests import model_docs


def offsets(queries):
    off = np.zeros(len(queries) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(q) for q in queries])
    return off


# ---- (a) the definition
def brute_len(docs, q):
    """len of every position of one query: the longest q[x, x + l) that some document contains."""
    out = []
    for x in range(len(q)):
        l = len(q) - x
        while l > 0 and not any(d.find(q[x:x + l]) >= 0 for d in docs):
            l -= 1
        out.append(l)
    return out


def brute_range(docs, g, s):
    """[start, end) of the ranks of g whose document suffix starts with s; (0, 0) for b"" or none."""
    text, starts = model_docs.concat(docs)
    n = len(text)
    if not s or n == 0:
        return 0, 0
    ends = np.append(starts[1:], n)
    hits = [i for i, p in enumerate(g.tolist())
            if text[p:int(ends[model_docs.doc_of(starts, p)])].startswith(s)]
    if not hits:
        return 0, 0
    assert hits == list(range(hits[0], hits[-1] + 1))
    return hits[0], hits[-1] + 1


def brute_smems(lens, min_len):
    """Offsets x of one query whose match [x, x + lens[x]) has min_len bytes or more and lies inside no
    other match of the query."""
    out = []
    for x, l in enumerate(lens):
        inside = any(y != x and y <= x and x + l <= y + m for y, m in enumerate(lens))
        if l >= min_len and not inside:
            out.append(x)
    return out


# ---- (b) the device steps
def _suffix(text, starts, n, p):
    d = model_docs.doc_of(starts, p)
    return text[p:int(starts[d + 1]) if d + 1 < len(starts) else n]


def _common(a, b, c):
    while c < len(a) and c < len(b) and a[c] == b[c]:
        c += 1
    return c


def search(text, starts, g, pat):
    """(len, witness rank) of one pattern: the binary search with the bounds' common-prefix lengths."""
    n = len(g)
    lo, hi, llo, lhi = 0, n, 0, 0                      # lo = the lower bound's rank + 1
    while lo < hi:
        mid = lo + (hi - lo) // 2
        s = _suffix(text, starts, n, int(g[mid]))
        c0 = min(llo, lhi)
        assert s[:c0] == pat[:c0]                      # the invariant that lets a probe start at c0
        c = _common(pat, s, c0)
        if c == len(pat):
            return c, mid
        if c < len(s) and pat[c] < s[c]:
            hi, lhi = mid, c
        else:
            lo, llo = mid + 1, c
    return (llo, lo - 1) if llo >= lhi else (lhi, hi)


def interval(lcp, w, l):
    """The LCP interval of depth l around rank w: [largest i <= w with lcp[i] < l, smallest i > w with
    lcp[i] < l, or n)."""
    s = w
    while lcp[s] >= l:
        s -= 1
    e = w + 1
    while e < len(lcp) and lcp[e] >= l:
        e += 1
    return s, e


def model(docs, g, glcp, queries):
    """(offsets, len, start, end) over all pattern positions, as the device entry points write them."""
    text, starts = model_docs.concat(docs)
    off = offsets(queries)
    qb = int(off[-1])
    ln, st, en = (np.zeros(qb, dtype=np.uint32) for _ in range(3))
    for k, q in enumerate(queries):
        for j in range(len(q)):
            x = int(off[k]) + j
            l, w = search(text, starts, g, q[j:]) if len(g) else (0, 0)
            ln[x] = l
            if l > 0:
                st[x], en[x] = interval(glcp, w, l)
    return off, ln, st, en


def smems(off, ln, min_len):
    """(offsets u64[nq + 1], qpos): the rule of b200sa_smems_dev."""
    nq = len(off) - 1
    out_off = np.zeros(nq + 1, dtype=np.uint64)
    qpos = []
    for k in range(nq):
        a, b = int(off[k]), int(off[k + 1])
        for x in range(a, b):
            if ln[x] >= min_len and (x == a or ln[x - 1] <= ln[x]):
                qpos.append(x - a)
        out_off[k + 1] = len(qpos)
    return out_off, np.asarray(qpos, dtype=np.uint32)
