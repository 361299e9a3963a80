"""Host statements of best hits (include/b200sa.h, B200SA_APPROX_BEST) over the plain definitions of
tests/model_approx.py (Hamming) and tests/model_edit.py (edit): (a) the definition -- best(q) the least distance of
q's occurrences within k, and q's list its occurrences with d(p) <= t(q) = min(k, best(q) + s) -- and (b) the
device's schedule: rounds t = 0 .. k over the live queries, best(q) the first round with an occurrence, the count
of q's last live round, then one emission per distinct t(q).  A single text is one document."""
import numpy as np

from tests import model_approx, model_edit

BRUTE = {"hamming": model_approx.brute, "edit": model_edit.brute}


def lists(packed):
    """Per-query lists of (p, d) of an (offsets, pos, dist) triple."""
    off, pos, dist = packed
    return [list(zip(pos[int(a):int(b)].tolist(), dist[int(a):int(b)].tolist())) for a, b in zip(off[:-1], off[1:])]


def best_of(docs, queries, k, metric):
    """best(q) of every query: the least d(p) of its occurrences within k, None without one."""
    return [min(d for _, d in h) if h else None for h in lists(BRUTE[metric](docs, queries, k))]


def threshold(best, k, s):
    """t(q) = min(k, best(q) + s), or None for a query with no occurrence."""
    return None if best is None else min(k, best + s)


def select(docs, queries, k, s, metric):
    """The definition: the occurrences within k, filtered to d(p) <= t(q) on the host."""
    out = []
    for h in lists(BRUTE[metric](docs, queries, k)):
        t = threshold(min(d for _, d in h), k, s) if h else -1
        out.append([(p, d) for p, d in h if d <= t])
    return model_approx._pack(out)


def rounds(docs, queries, k, s, metric):
    """The device's schedule: ((offsets, pos, dist), the number of rounds, the live queries of every round).  Round
    t counts the live queries at threshold t as one batch; a query is live while it has no occurrence yet or
    t <= best + s; the emission runs once per distinct final threshold over the queries that end there."""
    nq = len(queries)
    best, cnt, live_per_round = [None] * nq, [0] * nq, []
    for t in range(k + 1):
        live = [q for q in range(nq) if queries[q] and (best[q] is None or t <= best[q] + s)]
        if not live:
            break
        live_per_round.append(live)
        off = BRUTE[metric](docs, [queries[q] for q in live], t)[0]
        for i, q in enumerate(live):
            cnt[q] = int(off[i + 1] - off[i])
            if best[q] is None and cnt[q] > 0:
                best[q] = t
    out = [[] for _ in range(nq)]
    for t in sorted({threshold(b, k, s) for b in best if b is not None}):
        group = [q for q in range(nq) if best[q] is not None and threshold(best[q], k, s) == t]
        for q, h in zip(group, lists(BRUTE[metric](docs, [queries[q] for q in group], t))):
            assert len(h) == cnt[q], "an emission differs from its query's last count"
            out[q] = h
    assert [len(h) for h in out] == cnt
    return model_approx._pack(out), len(live_per_round), live_per_round
