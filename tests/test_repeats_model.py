"""The numpy model of the repeats (tests/model_repeats.py, the device formulation) against brute force
straight from the definitions in include/b200sa.h, and the facts that follow from the definitions."""
import itertools

import numpy as np

from tests import families, model_docs, model_repeats as mr


def _check(docs, lens):
    """Model == definition for rl, the runs and every mode's spans at every L of `lens`."""
    docs = [bytes(d) for d in docs]
    g, glcp = model_docs.brute(docs)
    text, starts = model_docs.concat(docs)
    n = len(text)
    assert np.array_equal(mr.repeat_lens(g, glcp), mr.brute_repeat_lens(docs)), docs
    rl = mr.repeat_lens(g, glcp)
    for L in lens:
        grams = {s: w for s, w in mr.brute_grams(docs, L).items() if len(w) > 1}
        start, end, first, last = mr.runs(g, glcp, L)
        # the runs are the distinct L-byte strings that occur twice, in the table's order
        assert len(start) == len(grams), (docs, L)
        seen = []
        for a, b, f, l in zip(start.tolist(), end.tolist(), first.tolist(), last.tolist()):
            s = text[int(g[a]):int(g[a]) + L]
            assert sorted(g[a:b].tolist()) == grams[s] and (f, l) == (grams[s][0], grams[s][-1]), (docs, L)
            seen.append(s)
        assert seen == sorted(grams), (docs, L)
        want = mr.brute_flags(docs, L)
        got = {m: mr.flags(g, glcp, starts if len(docs) else None, L, m) for m in mr.MODES} if len(docs) else \
              {m: np.zeros(0, dtype=bool) for m in mr.MODES}
        for m in mr.MODES:
            assert np.array_equal(got[m], want[m]), (docs, L, m)
            b, e, cov = mr.spans(got[m], starts, L)
            wb, we, wcov = mr.spans_of_flags(docs, want[m], L)
            assert np.array_equal(b, wb) and np.array_equal(e, we) and cov == wcov, (docs, L, m)
            assert cov == int((e.astype(np.int64) - b).sum()) and np.all(e - b >= L)
            assert np.all(b[1:] >= e[:-1])                              # ascending and disjoint
            d = np.searchsorted(starts, b, side="right") - 1           # every span inside one document
            assert np.all(e <= np.append(starts[1:], n)[d])
        # the facts under the definitions
        assert np.array_equal(got[mr.ANY], rl >= L)
        assert int((end.astype(np.int64) - start).sum()) == int(got[mr.ANY].sum())
        assert not np.any(got[mr.EARLIER_DOC] & ~got[mr.EARLIER]) and not np.any(got[mr.EARLIER] & ~got[mr.ANY])
        assert not np.any(got[mr.EARLIER_DOC] & ~got[mr.OTHER_DOC]) and not np.any(got[mr.OTHER_DOC] & ~got[mr.ANY])
        cover = np.zeros(n, dtype=bool)                                 # ANY covers the union of [p, p + rl[p])
        for p in np.nonzero(rl >= L)[0]:
            cover[p:p + int(rl[p])] = True
        b, e, _ = mr.spans(got[mr.ANY], None, L)
        mask = np.zeros(n, dtype=bool)
        for x, y in zip(b.tolist(), e.tolist()):
            mask[x:y] = True
        assert np.array_equal(mask, cover), (docs, L)
        if len(docs) == 1:                                              # one document is the single text
            for m in (mr.ANY, mr.EARLIER):
                assert np.array_equal(mr.flags(g, glcp, None, L, m), got[m])
            assert not got[mr.OTHER_DOC].any() and not got[mr.EARLIER_DOC].any()


def test_every_text_over_ab_up_to_length_8():
    for n in range(0, 9):
        for t in itertools.product(b"ab", repeat=n):
            _check([bytes(t)], range(1, 10))


def test_every_set_of_up_to_3_documents_over_ab_of_total_length_8():
    count = 0
    for n in range(0, 9):
        for t in itertools.product(b"ab", repeat=n):
            t = bytes(t)
            for i in range(n + 1):
                for j in range(i, n + 1):                    # empty documents at the front, middle and end
                    if n == 8 and (i + j) % 3:               # a third of the cuts of the longest texts
                        continue
                    _check([t[:i], t[i:j], t[j:]], (1, 2, 3, n, n + 1))
                    count += 1
                _check([t[:i], t[i:]], (1, 2, 3))
    assert count > 10_000


def test_random_document_sets():
    rng = np.random.default_rng(71)
    for _ in range(2000):
        docs = model_docs.random_docs(rng)
        _check(docs, (1, 2, 3, 5, 8))


def test_family_heads():
    texts = [bytes(t[:48]) for _, t in families.adversarial()] + [families.fib_word(40)]
    for t in texts:
        t = bytes(t)
        _check([t], (1, 2, 3, 8, len(t), len(t) + 1))
        _check([t[:11], b"", t[11:30], t[5:25]], (1, 2, 3, 8))


def test_touching_spans():
    # "abab": the grams at 0 and 2 touch inside one document and merge; as two documents they stay two
    for docs, want in (([b"abab"], [(0, 4)]), ([b"ab", b"ab"], [(0, 2), (2, 4)]), ([b"ab", b"", b"ab"], [(0, 2), (2, 4)])):
        g, glcp = model_docs.brute(docs)
        _, starts = model_docs.concat(docs)
        b, e, cov = mr.duplicate_spans(g, glcp, starts, 2, mr.ANY)
        assert list(zip(b.tolist(), e.tolist())) == want and cov == 4
    g, glcp = model_docs.brute([b"ab", b"ab"])
    b, e, cov = mr.duplicate_spans(g, glcp, np.asarray([0, 2]), 2, mr.EARLIER_DOC)
    assert (b.tolist(), e.tolist(), cov) == ([2], [4], 2)


def test_huge_min_len_is_plain_u32_arithmetic():
    g, glcp = model_docs.brute([b"aaaa"])
    assert mr.duplicate_spans(g, glcp, None, 0xFFFFFFFF, mr.ANY)[2] == 0
    assert len(mr.runs(g, glcp, 0xFFFFFFFF)[0]) == 0


def test_serial_c_statement_equals_model():
    from tests import repeats_check
    rng = np.random.default_rng(72)
    sets = [model_docs.random_docs(rng) for _ in range(300)]
    sets += [[bytes(t[:700]), b"", bytes(t[300:900])] for _, t in families.adversarial()]
    for docs in sets:
        g, glcp = model_docs.brute(docs)
        _, starts = model_docs.concat(docs)
        if len(g) == 0:
            continue
        for L in (1, 2, 3, 8, 40):
            assert all(np.array_equal(a, b) for a, b in zip(repeats_check.runs(g, glcp, L), mr.runs(g, glcp, L)))
            for m in mr.MODES:
                got, want = repeats_check.spans(g, glcp, starts, L, m), mr.duplicate_spans(g, glcp, starts, L, m)
                assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and got[2] == want[2]
            for m in (mr.ANY, mr.EARLIER):
                got, want = repeats_check.spans(g, glcp, None, L, m), mr.duplicate_spans(g, glcp, None, L, m)
                assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and got[2] == want[2]
