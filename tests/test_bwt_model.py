"""The Burrows-Wheeler transform's statements (tests/model_bwt.py) against each other, without a GPU: known
answers, the model of the device steps against the brute-force rotation sort, and the validity rule
against the exact set of images, exhaustively on small inputs."""
import itertools

import numpy as np
import pytest

from tests import model_bwt as mb, model_docs

KNOWN = {   # input: (bwt, term_rows, full L, r), by brute-force rotation sorting
    (b"banana",): (b"annbaa", [4], "annb$aa", 5),
    (b"abracadabra",): (b"ardrcaaaabb", [3], "ard$rcaaaabb", 8),
    (b"ab", b"", b"b"): (b"bba", [3, 1, 5], "b $1 b $0 a $2", 6),
}


def _show(L, k):
    syms = ["$" if kind == 0 and k == 1 else ("$%d" % v if kind == 0 else chr(v)) for kind, v in L]
    return "".join(syms) if k == 1 else " ".join(syms)


@pytest.mark.parametrize("docs", list(KNOWN))
def test_known_answers(docs):
    bwt, term_rows, full, r = KNOWN[docs]
    got = mb.brute(list(docs))
    assert (got[0], got[1], _show(got[2], len(docs)), got[3]) == (bwt, term_rows, full, r)
    g, _ = model_docs.brute(list(docs))
    fb, ft, fr = mb.forward(list(docs), g)
    assert (fb, ft.tolist(), fr) == (bwt, term_rows, r)
    assert mb.inverse_by_definition(bwt, term_rows) == list(docs)
    for s in (1, 2, 3, 64, 1000):
        assert mb.inverse(bwt, term_rows, s)[0] == list(docs)


def _random_docs(rng):
    kind = int(rng.integers(0, 4))
    k = int(rng.integers(1, 7))
    if kind == 0:                                              # all 256 byte values
        return [bytes(rng.integers(0, 256, int(rng.integers(0, 40)), dtype=np.uint8)) for _ in range(k)]
    if kind == 1:                                              # empty documents first, in the middle and last
        docs = [bytes(rng.choice(list(b"ab"), int(rng.integers(1, 9))).tolist()) for _ in range(k)]
        for at in (0, len(docs) // 2, len(docs)):
            docs.insert(at, b"")
        return docs
    if kind == 2:                                              # repeated documents and runs
        d = bytes(rng.choice(list(b"ACGT"), int(rng.integers(1, 10))).tolist())
        return [d] * k + [d[:2] * 3]
    return model_docs.random_docs(rng)


def test_model_against_brute_force():
    rng = np.random.default_rng(131)
    sets = [[b""], [b"", b""], [b"x"], [b"", b"x", b""], [b"\x00\xff\x00"], [bytes(range(256))]]
    sets += [_random_docs(rng) for _ in range(400)]
    for docs in sets:
        bwt, term_rows, _, r = mb.brute(docs)
        g, _ = model_docs.brute(docs)
        fb, ft, fr = mb.forward(docs, g)
        assert (fb, ft.tolist(), fr) == (bwt, term_rows, r), docs
        assert mb.inverse_by_definition(bwt, term_rows) == [bytes(d) for d in docs], docs
        for s in (1, 3, 64, len(bwt) + 1):
            got, rec = mb.inverse(bwt, term_rows, s)
            assert got == [bytes(d) for d in docs], (docs, s)
            assert rec["longest"] >= 1 and rec["rulers"] >= len(docs)
        _, rec = mb.inverse(bwt, term_rows, len(bwt) + 1)      # a spacing above n: the terminator rows alone
        assert rec["rulers"] == len(docs)


def test_single_text_primary_index():
    rng = np.random.default_rng(132)
    for _ in range(100):
        t = bytes(rng.choice(list(b"abc"), int(rng.integers(1, 30))).tolist())
        bwt, term_rows, _, _ = mb.brute([t])
        sa = sorted(range(len(t)), key=lambda p: t[p:])
        assert term_rows == [1 + sa.index(0)]                   # 1 + the rank of position 0
        assert bwt == t[-1:] + bytes(t[p - 1] for p in sa if p > 0)   # row 0 is $t, then the suffix order


def _images(n, k):
    """The set of (bwt, term_rows) images of every k documents over {a, b} with n bytes in all."""
    out = set()
    for cuts in itertools.combinations_with_replacement(range(n + 1), k - 1):
        bounds = (0,) + cuts + (n,)
        for word in itertools.product(b"ab", repeat=n):
            w = bytes(word)
            docs = [w[bounds[i]:bounds[i + 1]] for i in range(k)]
            bwt, term_rows, _, _ = mb.brute(docs)
            out.add((bwt, tuple(term_rows)))
    return out


@pytest.mark.parametrize("k,nmax", [(1, 7), (2, 5), (3, 5)])
def test_validity_rule_is_exactly_the_images(k, nmax):
    """Every bwt over {a, b} and every term_rows (repeats and all) up to the sizes: the rule and the model
    accept exactly the images of some documents, and decode them to documents with that image."""
    for n in range(nmax + 1):
        images = _images(n, k)
        for word in itertools.product(b"ab", repeat=n):
            bwt = bytes(word)
            for term_rows in itertools.product(range(n + k), repeat=k):
                docs = mb.inverse_by_definition(bwt, term_rows)
                want = (bwt, tuple(term_rows)) in images
                assert (docs is not None) == want, (bwt, term_rows)
                got, rec = mb.inverse(bwt, term_rows, 2)
                assert got == docs, (bwt, term_rows)
                if want:
                    assert mb.brute(docs)[:2] == (bwt, list(term_rows))
                else:
                    assert rec["reject"] == ("terms" if len(set(term_rows)) < k else "cycles")
