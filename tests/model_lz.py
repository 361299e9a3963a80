"""Host statements of the longest previous factor and the LZ77 factorization (include/b200sa.h,
b200sa_lpf_dev, b200sa_lz77_dev): the definitions by brute force on the documents themselves (no suffix
array), and a numpy model of the device formulation (suffix_b200/csrc/lz.cuh) on the table and its LCP
array."""
import numpy as np

from tests import model_docs

LITERAL = 0xFFFFFFFF


def _docs(docs):
    return [docs] if isinstance(docs, (bytes, bytearray)) else list(docs)


# ------------------------------------------------------------------ the definitions
def brute_lpf(docs):
    """lpf[p]: the longest prefix of S_p that is a prefix of S_q for some q < p (S cut at document ends)."""
    text, starts = model_docs.concat(_docs(docs))
    n = len(text)
    ends = [int(x) for x in starts[1:]] + [n]
    de = [ends[model_docs.doc_of(starts, p)] for p in range(n)]
    lpf = np.zeros(n, dtype=np.uint32)
    for p in range(n):
        for q in range(p):
            k = 0
            while p + k < de[p] and q + k < de[q] and text[p + k] == text[q + k]:
                k += 1
            lpf[p] = max(lpf[p], k)
    return lpf


def serial_parse(lpf):
    """(start, length) of the greedy parse: f_0 = 0, f_(i+1) = f_i + max(1, lpf[f_i])."""
    n, p, starts = len(lpf), 0, []
    while p < n:
        starts.append(p)
        p += max(1, int(lpf[p]))
    starts = np.asarray(starts, dtype=np.uint32)
    return starts, np.maximum(np.asarray(lpf, dtype=np.uint32)[starts], 1).astype(np.uint32)


def decode(n, start, length, src, literal_bytes):
    """Rebuild the text from the factors, byte by byte (a copy may overlap its own output); literal_bytes
    holds one byte per literal, in factor order."""
    out = bytearray(n)
    lit = iter(literal_bytes)
    pos = 0
    for s, l, q in zip(start.tolist(), length.tolist(), src.tolist()):
        assert s == pos, (s, pos)
        if q == LITERAL:
            assert l == 1
            out[s] = next(lit)
        else:
            assert q < s
            for k in range(l):
                out[s + k] = out[q + k]
        pos = s + l
    assert pos == n
    return bytes(out)


# ------------------------------------------------------------------ the device formulation
def nearest_smaller(R):
    """(psv, nsv) over the values of R by one stack each; -1 / n where absent."""
    n = len(R)
    psv, nsv = np.full(n, -1, dtype=np.int64), np.full(n, n, dtype=np.int64)
    st = []
    for r in range(n):
        while st and R[st[-1]] > R[r]:
            nsv[st.pop()] = r
        psv[r] = st[-1] if st else -1
        st.append(r)
    return psv, nsv


def lpf_src(R, lam):
    """(lpf, src) in text order, as k_lz_lpf: ranges of lam between a rank and its psv / nsv."""
    R, lam = np.asarray(R, dtype=np.int64), np.asarray(lam, dtype=np.int64)
    n = len(R)
    psv, nsv = nearest_smaller(R)
    lpf = np.zeros(n, dtype=np.uint32)
    src = np.full(n, LITERAL, dtype=np.uint32)
    for r in range(n):
        a, b, p = psv[r], nsv[r], R[r]
        lL = int(lam[a + 1:r + 1].min()) if a >= 0 else 0
        lR = int(lam[r + 1:b + 1].min()) if b < n else 0
        lpf[p] = max(lL, lR)
        if lL >= lR and lL > 0:
            src[p] = R[a]
        elif lR > 0:
            src[p] = R[b]
    return lpf, src


def parse(lpf):
    """(marks bool[n], rounds) by path doubling, as k_lz_next / k_lz_mark / k_lz_square: a round marks
    J[p] for every marked p with J[p] < n, then squares J; the round that finds J[0] >= n does nothing."""
    lpf = np.asarray(lpf, dtype=np.int64)
    n = len(lpf)
    J = np.append(np.arange(n) + np.maximum(lpf, 1), n)
    marks = np.zeros(n, dtype=bool)
    if n:
        marks[0] = True
    rounds = 0
    for _ in range(n.bit_length()):
        if J[0] >= n:
            break
        q = J[np.nonzero(marks)[0]]
        marks[q[q < n]] = True
        J = J[J]
        rounds += 1
    return marks, rounds


def factors(R, lam):
    """(start, length, source, rounds): LPF, the doubling parse and the emit at the marks."""
    lpf, src = lpf_src(R, lam)
    marks, rounds = parse(lpf)
    start = np.nonzero(marks)[0].astype(np.uint32)
    return start, np.maximum(lpf[start], 1).astype(np.uint32), src[start], rounds
