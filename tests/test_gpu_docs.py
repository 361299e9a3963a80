"""The separator-free generalized suffix array (b200sa_docs_build[_dev], b200sa_docs_positions_dev,
suffix_b200.DocumentSuffixTable) against the definition: a Python brute force on small document
sets, SuffixTable on single documents, and the C checker of tests/docs_check.c at scale."""
import os

import numpy as np
import pytest
import torch

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen
from tests import docs_check, model_docs

pytestmark = pytest.mark.gpu

BAD_ARG = -1


def _u8(t) -> bytes:
    return t if isinstance(t, bytes) else np.ascontiguousarray(t, dtype=np.uint8).tobytes()


class _two_stage_sort:
    """Forces the two-stage sort of the crossing suffixes (by document, then by (lo, r))."""

    def __enter__(self):
        os.environ["B200SA_DOCS_SORT2"] = "1"

    def __exit__(self, *a):
        del os.environ["B200SA_DOCS_SORT2"]


def _check_brute(docs):
    st = DocumentSuffixTable(docs)
    g, lcp = model_docs.brute(docs)
    assert np.array_equal(st.table(), g), docs
    assert np.array_equal(st.lcp_lens(), lcp), docs
    return st


def _families(rng):
    out = [[], [b""], [b"", b"", b""], [b"x"], [b"", b"x"], [b"x", b""], [b"", b"", b"q", b""],
           [b"ab"], [b"a", b"b"], [b"b", b"a"], [b"a", b"a"]]
    for k in range(40):                                           # empty documents among others
        out.append([b"" if rng.random() < 0.5 else bytes(rng.choice(list(b"ab"), int(rng.integers(1, 6))))
                    for _ in range(int(rng.integers(1, 8)))])
    for k in range(40):                                           # duplicated documents
        d = bytes(rng.choice(list(b"ACGT"), int(rng.integers(1, 12))))
        out.append([d] * int(rng.integers(2, 9)) + [bytes(rng.choice(list(b"ACGT"), 5))])
    for k in range(40):                                           # documents that are prefixes of others
        d = bytes(rng.choice(list(b"abc"), int(rng.integers(2, 15))))
        cuts = sorted(int(x) for x in rng.integers(0, len(d) + 1, int(rng.integers(2, 6))))
        out.append([d[:c] for c in cuts] + [d])
    for k in range(40):                                           # one-byte runs
        out.append([bytes([int(rng.integers(0, 3))]) * int(rng.integers(1, 20)) for _ in range(int(rng.integers(1, 6)))])
    for k in range(20):                                           # all 256 byte values, 0x00 included
        allb = bytes(int(x) for x in rng.permutation(256))
        cut = sorted(int(x) for x in rng.integers(0, 256, 3))
        out.append([allb[:cut[0]], allb[cut[0]:cut[1]], allb[cut[1]:], bytes([0, 0, 255, 0])])
    for k in range(20):                                           # k = 1
        out.append([bytes(rng.choice(list(b"ab\x00"), int(rng.integers(1, 40))))])
    for k in range(100):
        out.append(model_docs.random_docs(rng))
    return out


def test_brute_force_families():
    rng = np.random.default_rng(11)
    sets = _families(rng)
    assert len(sets) >= 300
    for docs in sets:
        _check_brute(docs)


def test_brute_force_two_stage_sort():
    rng = np.random.default_rng(12)
    with _two_stage_sort():
        for docs in _families(rng)[::3]:
            _check_brute(docs)


def test_table_without_lcp():
    ctx = _lib.Context(0)
    rng = np.random.default_rng(13)
    for _ in range(30):
        docs = model_docs.random_docs(rng)
        text, starts = model_docs.concat(docs)
        g, lcp = ctx.docs_build(np.frombuffer(text, np.uint8), starts, with_lcp=False)
        assert lcp is None
        assert np.array_equal(g, model_docs.brute(docs)[0])
    ctx.close()


SINGLE = {
    "dna": lambda: _u8(gen.dna(1_000_000)),
    "english": lambda: _u8(gen.english(200_000)),
    "bytes": lambda: _u8(gen.rand_bytes(200_000)),
    "fixture10k": lambda: _u8(gen.fixture("AP009048_10000.fasta")),
    "fixture100k": lambda: _u8(gen.fixture("AP009048_100000.fasta")),
}


@pytest.mark.parametrize("name", list(SINGLE))
def test_single_document_is_the_suffix_table(name):
    t = SINGLE[name]()
    st = DocumentSuffixTable([t])
    ref = SuffixTable(t)
    assert np.array_equal(st.table(), ref.table())
    assert np.array_equal(st.lcp_lens(), ref.lcp_lens())


def _check_scale(docs):
    st = DocumentSuffixTable(docs)
    assert docs_check.check(st.text(), st.doc_starts(), st.table(), st.lcp_lens()) == 0
    return st


def test_scale_dna_cut_with_duplicates():
    rng = np.random.default_rng(21)
    t = _u8(gen.dna(4 << 20))
    cuts = np.unique(rng.integers(1, len(t), 3000))
    docs = [t[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(t)])]
    for k in rng.integers(0, len(docs), 40):                     # duplicated documents, placed anywhere
        docs.insert(int(rng.integers(0, len(docs) + 1)), docs[int(k)])
    docs.insert(5, b"")
    _check_scale(docs)


def test_scale_acgt_copies():
    docs = [b"ACGT"] * 100_000
    st = _check_scale(docs)
    # every T = "ACGT" suffix sorts by document: G lists the copies in order
    assert np.array_equal(st.table()[:100_000], np.arange(0, 400_000, 4, dtype=np.uint32))
    with _two_stage_sort():
        st2 = DocumentSuffixTable(docs)
    assert np.array_equal(st2.table(), st.table()) and np.array_equal(st2.lcp_lens(), st.lcp_lens())


def test_scale_fixture_lines():
    lines = _u8(gen.fixture("AP009048_100000.fasta")).split(b"\n")
    _check_scale(lines)


def test_scale_wide_keys_take_the_two_stage_sort():
    # n = 2^22, one document of 2^21 bytes and 2^21 one-byte documents: (lo, r, d) needs 66 bits
    docs = [_u8(gen.dna(1 << 21))] + [bytes([b]) for b in _u8(gen.dna(1 << 21))]
    _check_scale(docs)


# ---- queries
def _brute_positions(docs, q):
    out = []
    for d, doc in enumerate(docs):
        i = doc.find(q)
        while i >= 0:
            out.append((d, i))
            i = doc.find(q, i + 1)
    return out


def test_queries_against_brute_force():
    rng = np.random.default_rng(31)
    alpha = b"ACG\x00"
    docs = [bytes(alpha[int(c)] for c in rng.integers(0, 4, int(rng.integers(0, 900)))) for _ in range(24)]
    docs += [docs[3], docs[7][:50], b"", b"\x00\x00\x00"]
    st = DocumentSuffixTable(docs)
    text, starts = st.text(), st.doc_starts()
    nonempty = [d for d in range(len(docs)) if docs[d]]
    qs, kinds = [], []
    for k in range(50_000):
        r = k % 4
        if r == 0:                                               # substrings of documents
            d = docs[nonempty[int(rng.integers(0, len(nonempty)))]]
            a = int(rng.integers(0, len(d)))
            qs.append(d[a:a + int(rng.integers(1, 14))])
        elif r == 1:                                             # strings spanning a boundary in C
            d = int(rng.integers(1, len(docs)))
            s = int(starts[d])
            if s == 0 or s >= len(text):
                s = int(starts[nonempty[1]])
            qs.append(text[max(0, s - int(rng.integers(1, 8))):s + int(rng.integers(1, 8))])
        elif r == 2:                                             # random strings
            qs.append(bytes(alpha[int(c)] for c in rng.integers(0, 4, int(rng.integers(1, 10)))))
        else:                                                    # strings containing 0x00
            q = bytearray(bytes(alpha[int(c)] for c in rng.integers(0, 4, int(rng.integers(1, 8)))))
            q[int(rng.integers(0, len(q)))] = 0
            qs.append(bytes(q))
        kinds.append(r)
    qs.append(b"")
    kinds.append(-1)
    s_arr, e_arr = st.positions_batch(qs)
    g = st.table()
    spanning_empty = 0
    for q, kind, s, e in zip(qs, kinds, s_arr, e_arr):
        want = sorted(_brute_positions(docs, q)) if q else []
        p = g[s:e].astype(np.int64)
        d = np.searchsorted(starts, p, side="right") - 1
        got = sorted(zip(d.tolist(), (p - starts[d]).tolist()))
        assert got == want, (q, kind)
        spanning_empty += kind == 1 and not want
    assert spanning_empty > 1000       # most strings across a document end occur nowhere inside one
    # the host path agrees on a sample, and the single-query API
    for q in qs[:2000:7]:
        want = sorted(_brute_positions(docs, q))
        rows = st.positions(q)
        assert sorted(map(tuple, rows.tolist())) == want
        assert st.contains(q) == bool(want)
        ap = st.any_position(q)
        assert (ap is None) == (not want) and (ap is None or tuple(ap) in want)
    assert st.any_position(b"") is None and len(st.positions(b"")) == 0 and not st.contains(b"")
    # positions come in table order
    rows = st.positions(b"A")
    assert np.array_equal(st.doc_starts()[rows[:, 0]] + rows[:, 1], g[st._range(b"A")[0]:st._range(b"A")[1]])


def test_accessors_and_locate():
    docs = [b"banana", b"", b"ana", b"nab"]
    st = DocumentSuffixTable(docs)
    assert len(st) == st.len() == 12 and not st.is_empty()
    assert st.doc_starts().tolist() == [0, 6, 6, 9]
    got = [(st.suffix_bytes(i), int(st.locate([st.table()[i]])[0, 0])) for i in range(len(st))]
    assert got == sorted((d[o:], k) for k, d in enumerate(docs) for o in range(len(d)))
    assert st.locate([0, 5, 6, 8, 9, 11]).tolist() == [[0, 0], [0, 5], [2, 0], [2, 2], [3, 0], [3, 2]]
    e = DocumentSuffixTable([])
    assert e.is_empty() and len(e.table()) == 0 and e.positions(b"a").shape == (0, 2)
    assert e.any_position(b"a") is None
    s, t = e.positions_batch([b"a", b""])
    assert s.tolist() == [0, 0] and t.tolist() == [0, 0]
    one = DocumentSuffixTable([b"", b"z", b""])
    assert one.table().tolist() == [0] and one.lcp_lens().tolist() == [0]
    assert one.any_position(b"z") == (1, 0)


# ---- device entry
def _dev_build(ctx, text: bytes, starts, with_lcp=True):
    n = len(text)
    d_t = torch.from_numpy(np.frombuffer(text or b"\0", np.uint8).copy()).cuda()
    s = np.asarray(starts, dtype=np.uint32)
    d_s = torch.from_numpy(s.view(np.int32).copy() if len(s) else np.zeros(1, np.int32)).cuda()
    d_g = torch.full((max(n, 1),), -1, dtype=torch.int32, device="cuda")
    d_l = torch.full((max(n, 1),), -1, dtype=torch.int32, device="cuda")
    ctx.docs_build_dev(d_t.data_ptr(), n, d_s.data_ptr(), len(s), d_g.data_ptr(), d_l.data_ptr() if with_lcp else 0,
                       torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return d_g.cpu().numpy().view(np.uint32)[:n], d_l.cpu().numpy().view(np.uint32)[:n]


def test_device_entry_equals_host_entry():
    ctx = _lib.Context(0)
    rng = np.random.default_rng(41)
    sets = [model_docs.random_docs(rng) for _ in range(40)]
    t = _u8(gen.dna(300_001))
    sets.append([t[:1000], t[1000:1001], b"", t[1001:200_000], t[1000:1001], t[200_000:]])
    sets += [[b"x"], [b"", b"x", b""], [], [b""]]
    for docs in sets:
        text, starts = model_docs.concat(docs)
        g, lcp = ctx.docs_build(np.frombuffer(text, np.uint8), starts)
        dg, dl = _dev_build(ctx, text, starts)
        assert np.array_equal(g, dg) and np.array_equal(lcp, dl), docs
        dg2, _ = _dev_build(ctx, text, starts, with_lcp=False)
        assert np.array_equal(g, dg2)
    # an unaligned device text takes the build's aligned copy
    text, starts = model_docs.concat(sets[-5])
    d_t = torch.from_numpy(np.frombuffer(b"?" + text, np.uint8).copy()).cuda()
    d_s = torch.from_numpy(starts.view(np.int32).copy()).cuda()
    d_g = torch.empty(len(text), dtype=torch.int32, device="cuda")
    ctx.docs_build_dev(d_t.data_ptr() + 1, len(text), d_s.data_ptr(), len(starts), d_g.data_ptr(), 0,
                       torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(d_g.cpu().numpy().view(np.uint32), ctx.docs_build(np.frombuffer(text, np.uint8), starts)[0])
    ctx.set_timing(True)
    _dev_build(ctx, text, starts)
    names = [p for p, _ in ctx.phase_times()]
    ctx.set_timing(False)
    for p in ("docs_check", "docs_split", "docs_sort", "docs_place", "docs_fill", "docs_out"):
        assert p in names, names
    ctx.close()


BAD_STARTS = {
    "first_not_zero": (b"abcdef", [1, 3]),
    "not_ascending": (b"abcdef", [0, 4, 2]),
    "above_n": (b"abcdef", [0, 3, 7]),
    "no_docs": (b"abcdef", []),
    "n1_first_not_zero": (b"a", [1]),
    "n0_above_n": (b"", [0, 1]),
}


@pytest.mark.parametrize("name", list(BAD_STARTS))
def test_bad_doc_starts(name):
    text, starts = BAD_STARTS[name]
    ctx = _lib.Context(0)
    with pytest.raises(_lib.B200SAError) as e:
        ctx.docs_build(np.frombuffer(text, np.uint8), np.asarray(starts, np.uint32))
    assert e.value.code == BAD_ARG and "doc_starts" in str(e.value)
    with pytest.raises(_lib.B200SAError) as e:
        _dev_build(ctx, text, starts)
    assert e.value.code == BAD_ARG and "doc_starts" in str(e.value)
    # the context stays usable
    g, _ = ctx.docs_build(np.frombuffer(b"abab", np.uint8), np.asarray([0, 2], np.uint32))
    assert g.tolist() == [0, 2, 1, 3]
    ctx.close()


def test_concurrent_with_suffix_table():
    # DocumentSuffixTable and SuffixTable share the default context: builds from two threads at once
    # must give the same arrays as builds one after the other
    import threading
    docs = [_u8(gen.dna(300_000, seed=s)) for s in (1, 2)] + [b"ACGT" * 5000]
    t = _u8(gen.english(400_000))
    want_d = DocumentSuffixTable(docs)
    want_t = SuffixTable(t).table()
    errors = []

    def run(fn):
        try:
            for _ in range(6):
                fn()
        except Exception as e:               # reported in the main thread
            errors.append(e)

    def build_docs():
        st = DocumentSuffixTable(docs)
        assert np.array_equal(st.table(), want_d.table()) and np.array_equal(st.lcp_lens(), want_d.lcp_lens())

    def build_table():
        assert np.array_equal(SuffixTable(t).table(), want_t)

    th = [threading.Thread(target=run, args=(f,)) for f in (build_docs, build_table)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
