"""Best hits of approximate positions (tests/model_best.py) against the plain definitions, exhaustively over small
texts on {a, b}: the identity "the BEST list is the plain list at t(q)", the s = 0, s >= k and k = 0 properties, and
the round schedule the device runs.  CPU only."""
import itertools

import numpy as np
import pytest

from suffix_b200 import _approx
from tests import model_best

METRICS = ("hamming", "edit")


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def _words(lengths):
    return [bytes(w) for m in lengths for w in itertools.product(b"ab", repeat=m)]


QUERIES = _words(range(4))                            # b"" and every word of 1 to 3 letters


def _sets():
    """Every text on {a, b} of at most 5 letters as one text, and cut into documents around an empty one."""
    out = []
    for text in _words(range(6)):
        out.append([text])
        if text:
            cut = len(text) // 2
            out.append([text[:cut], b"", text[cut:]])
    return out


@pytest.mark.parametrize("metric", METRICS)
def test_best_list_is_the_plain_list_at_its_threshold(metric):
    for docs in _sets():
        plain = {k: model_best.lists(model_best.BRUTE[metric](docs, QUERIES, k)) for k in range(5)}
        for k in range(5):
            best = model_best.best_of(docs, QUERIES, k, metric)
            for s in range(4):
                got = model_best.lists(model_best.select(docs, QUERIES, k, s, metric))
                for q, b in enumerate(best):
                    t = model_best.threshold(b, k, s)
                    assert got[q] == (plain[t][q] if t is not None else []), (docs, QUERIES[q], k, s)
                    if s == 0:
                        assert all(d == b for _, d in got[q])
                    if s >= k:
                        assert got[q] == plain[k][q]
                    if k == 0:
                        assert got[q] == plain[0][q]


@pytest.mark.parametrize("metric", METRICS)
def test_round_schedule_yields_the_definition(metric):
    for docs in _sets():
        for k in range(5):
            best = model_best.best_of(docs, QUERIES, k, metric)
            for s in range(4):
                got, nrounds, live = model_best.rounds(docs, QUERIES, k, s, metric)
                assert _same(got, model_best.select(docs, QUERIES, k, s, metric)), (docs, k, s)
                ends = [model_best.threshold(b, k, s) for b in best]
                want = max([k if e is None else e for q, e in enumerate(ends) if QUERIES[q]], default=-1) + 1
                assert nrounds == want, (docs, k, s)
                for t, lv in enumerate(live):              # live in round t: nothing found yet, or t <= best + s
                    assert lv == [q for q, b in enumerate(best) if QUERIES[q] and (b is None or t <= b + s)]


def test_rounds_on_reads_stop_at_their_best():
    rng = np.random.default_rng(61)
    text = bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), 3000))
    qs = []
    for e in range(5):
        a = int(rng.integers(0, 2950))
        q = bytearray(text[a:a + 40])
        for x in rng.choice(40, e, replace=False).tolist():
            q[x] = ord("N")
        qs.append(bytes(q))
    for metric in METRICS:
        got, nrounds, live = model_best.rounds([text], qs, 8, 0, metric)
        assert _same(got, model_best.select([text], qs, 8, 0, metric))
        best = model_best.best_of([text], qs, 8, metric)
        assert best == [0, 1, 2, 3, 4] if metric == "hamming" else all(b <= e for b, e in zip(best, range(5)))
        assert nrounds == max(best) + 1
        assert [len(x) for x in live] == [sum(b >= t for b in best) for t in range(nrounds)]


def test_python_best_argument():
    assert _approx._flags(None) == 0
    assert _approx._flags(0) == 0x100000
    assert _approx._flags(31) == _approx._flags(np.int64(31)) == 0x100000 | (31 << 8)
    for bad in (True, False, np.bool_(True), -1, 32, 1.0, "1"):
        with pytest.raises(ValueError):
            _approx._flags(bad)
