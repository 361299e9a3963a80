"""The approximate document listing (B200SA_APPROX_DOCUMENTS on b200sa_docs_approx_positions_dev, the
approximate_documents* methods of DocumentSuffixTable), for all 16 mixes of the edit metric, best hits, IUPAC
queries and both strands: against tests/model_approx_docs.py on small collections, against the call without the
flag grouped on the host on large ones, against documents_batch at threshold 0, and the listing protocol, the
edge cases and the argument errors."""
import numpy as np
import pytest

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen
from tests import model_approx_docs, model_docs, model_strand
from tests.test_gpu_approx import MARK, _abi, _fetch, _same
from tests.test_gpu_approx import _queries as _plain_queries
from tests.test_gpu_docs import _families, _u8
from tests.test_gpu_edit import _reads
from tests.test_gpu_iupac import _guides, _masked_dna
from tests.test_gpu_iupac import _queries as _iupac_queries
from tests.test_gpu_strand import _dna_queries

pytestmark = pytest.mark.gpu

BAD_ARG = -1
EDIT = 0x10000                                  # B200SA_APPROX_EDIT
BEST = 0x100000                                 # B200SA_APPROX_BEST
IUPAC = 0x1000000                               # B200SA_APPROX_IUPAC
BOTH = 0x10000000                               # B200SA_APPROX_BOTH_STRANDS
DOCS = 0x20000000                               # B200SA_APPROX_DOCUMENTS
MINUS = model_strand.MINUS
METRIC = {"hamming": 0, "edit": EDIT}
MIXES = [(metric, iupac, best, strands) for metric in ("hamming", "edit") for iupac in (False, True)
         for best in (None, 1) for strands in ("forward", "both")]


def _kf(k, metric, iupac, best, strands, docs=True):
    return (k | METRIC[metric] | (IUPAC if iupac else 0) | (0 if best is None else (best << 8) | BEST) |
            (BOTH if strands == "both" else 0) | (DOCS if docs else 0))


def _packed(res, strands):
    """(offsets, values, d | MINUS) of what a method returns for strands=."""
    if strands == "forward":
        return res
    off, val, dist, minus = res
    assert dist.dtype == np.uint32 and minus.dtype == bool and not (dist & MINUS).any()
    return off, val, dist | np.where(minus, np.uint32(MINUS), np.uint32(0))


@pytest.mark.parametrize("metric,iupac,best,strands", MIXES)
def test_families_equal_model(metric, iupac, best, strands):
    rng = np.random.default_rng(400 + MIXES.index((metric, iupac, best, strands)))
    sets = _families(rng)[::4] + [[_masked_dna(rng, int(rng.integers(1, 120))) for _ in range(4)] for _ in range(8)]
    ctx = _lib.Context(0)
    for i, docs in enumerate(sets):
        k = [0, 1, 2, 3, 4, 31][i % 6]
        if iupac:
            qs = _iupac_queries(rng, docs, k)
        else:
            qs = _plain_queries(rng, docs, k) if i % 2 else _dna_queries(rng, docs, k)
        g, _ = model_docs.brute(docs)
        text, starts = model_docs.concat(docs)
        want = model_approx_docs.brute(docs, qs, k, metric, iupac, best, strands)
        assert _same(_fetch(ctx, text, g, qs, _kf(k, metric, iupac, best, strands), starts), want), (docs, k)
        st = DocumentSuffixTable(docs)
        kw = dict(metric=metric, iupac=iupac, best=best, strands=strands)
        assert _same(_packed(st.approximate_documents_batch(qs, k, **kw), strands), want), (docs, k)
        freq = st.approximate_document_frequencies(qs, k, **kw)
        assert freq.dtype == np.uint32 and np.array_equal(freq, np.diff(want[0].astype(np.int64))), (docs, k)
        _, one, dist = _packed((None,) + tuple(st.approximate_documents(qs[-1], k, **kw)), strands)
        a, b = int(want[0][-2]), int(want[0][-1])
        assert np.array_equal(one, want[1][a:b]) and np.array_equal(dist, want[2][a:b]), (docs, k)
    ctx.close()


def _copies(base, count, rng, sub, indel):
    """count copies of base, each with substitutions at rate sub and single-byte insertions or deletions at rate
    indel."""
    bases = np.frombuffer(b"ACGT", dtype=np.uint8)
    out = []
    for _ in range(count):
        c = base.copy()
        s = rng.random(len(c)) < sub
        c[s] = rng.choice(bases, int(s.sum()))
        at = np.flatnonzero(rng.random(len(c)) < indel)
        ins = rng.random(len(at)) < 0.5
        c = np.insert(c, at[ins], rng.choice(bases, int(ins.sum())))
        c = np.delete(c, at[~ins] + np.searchsorted(at[ins], at[~ins], side="right"))
        out.append(c.tobytes())
    return out


@pytest.fixture(scope="module")
def collections():
    """(name, documents, reads, guides + NGG): 10^7 bases in ~1 kB documents, and 100 mutated copies of one
    100 kB genome."""
    rng = np.random.default_rng(410)
    t = gen.dna(10_000_000)
    text = _u8(t)
    cuts = np.unique(rng.integers(1, len(t), 10_000))
    kb = [text[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(t)])]
    reads = _reads(t, rng, 10_000, 150, 0.01, 0.005)
    reads = [model_strand.revcomp(r) if i % 2 else r for i, r in enumerate(reads)]
    guides = [g for g in _guides(t, rng, 1000) if g.endswith(b"NGG")]
    base = gen.dna(100_000)
    pan = _copies(base, 100, rng, 0.01, 0.001)
    pan_reads = []
    for i in range(10_000):
        c = np.frombuffer(pan[int(rng.integers(0, len(pan)))], dtype=np.uint8)
        r = _reads(c, rng, 1, 150, 0.005, 0.002)[0]
        pan_reads.append(model_strand.revcomp(r) if i % 2 else r)
    pan_guides = [g for g in _guides(base, rng, 1000) if g.endswith(b"NGG")]
    return [("kb_documents", DocumentSuffixTable(kb), reads, guides),
            ("mutated_copies", DocumentSuffixTable(pan), pan_reads, pan_guides)]


@pytest.mark.parametrize("metric,iupac,best,strands", MIXES)
def test_large_collections_equal_the_flagless_call_grouped(collections, metric, iupac, best, strands):
    kw = dict(metric=metric, iupac=iupac, best=best, strands=strands)
    for name, st, reads, guides in collections:
        qs, k = (guides, 3 if metric == "hamming" else 2) if iupac else (reads, 4 if metric == "hamming" else 3)
        hits = _packed(st.approximate_positions_batch(qs, k, **kw), strands)
        want = model_approx_docs.group(hits, st.doc_starts())
        got = _packed(st.approximate_documents_batch(qs, k, **kw), strands)
        assert _same(got, want), name
        assert np.array_equal(st.approximate_document_frequencies(qs, k, **kw), np.diff(want[0].astype(np.int64)))
        n_docs, n_hits = int(want[0][-1]), int(hits[0][-1])
        assert 0 < n_docs <= n_hits, name
        if name == "mutated_copies" and best is None and strands == "both":     # most reads land in most copies
            assert n_docs >= 10 * len(qs) and (n_hits > n_docs or metric == "hamming"), (name, n_docs, n_hits)
        if strands == "both" and not iupac:                                     # half the reads are on the minus strand
            assert (got[2] & MINUS).any() and not (got[2] & MINUS).all(), name


def test_threshold_zero_equals_documents_batch():
    rng = np.random.default_rng(420)
    t = gen.dna(300_000)
    text = _u8(t)
    cuts = np.unique(rng.integers(1, len(t), 300))
    docs = [text[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(t)])]
    docs[5] = b""
    st = DocumentSuffixTable(docs + [docs[3], docs[7][:40]])
    qs = [bytes(text[a:a + int(m)]) for a, m in zip(rng.integers(0, len(t) - 20, 400), rng.integers(1, 20, 400))]
    qs += [b"", b"A", b"ACGT", docs[3], docs[3] + b"A"]
    off, ds, cnt = st.documents_batch(qs)
    got = st.approximate_documents_batch(qs, 0)
    assert np.array_equal(got[0], off) and np.array_equal(got[1], ds) and not got[2].any()
    assert np.array_equal(st.approximate_document_frequencies(qs, 0), st.document_frequencies(qs))


def test_cap_protocol_and_null_distances():
    rng = np.random.default_rng(430)
    text = _masked_dna(rng, 3000)
    starts = np.array([0, 400, 400, 1000, 1013, 2200], dtype=np.uint32)
    docs = [text[a:b] for a, b in zip(starts, list(starts[1:]) + [len(text)])]
    g = DocumentSuffixTable(docs).table()
    up = text.upper()
    qs = [bytes(b if b in b"ACGT" else 65 for b in up[a:a + 10]) for a in rng.integers(0, 2990, 20)]
    qs = qs + [model_strand.revcomp(q) for q in qs[:4]] + [b"GAATTC", b"", b"AN", b"AC"]
    ctx = _lib.Context(0)
    for metric, iupac, best, strands in MIXES:
        kf = _kf(2, metric, iupac, best, strands)
        want = model_approx_docs.brute(docs, qs, 2, metric, iupac, best, strands)
        total = int(want[0][-1])
        assert total > 1
        for cap in (0, 1, total - 1):                                        # offsets only
            tot, off, pos, dist = _abi(ctx, text, g, qs, kf, cap, starts, buf=total + 5)
            assert tot == total and np.array_equal(off, want[0])
            assert (pos == MARK).all() and (dist == MARK).all(), cap
        tot, off, pos, dist = _abi(ctx, text, g, qs, kf, total, starts, buf=total + 5)   # fits: nothing past total
        assert tot == total and np.array_equal(off, want[0])
        assert np.array_equal(pos[:total], want[1]) and np.array_equal(dist[:total], want[2])
        assert (pos[total:] == MARK).all() and (dist[total:] == MARK).all()
        tot, off, pos, _ = _abi(ctx, text, g, qs, kf, total + 5, starts, with_mis=False, buf=total + 5)
        assert tot == total and np.array_equal(pos[:total], want[1]) and (pos[total:] == MARK).all()
    ctx.close()


def test_nq0_n0_and_repeated_calls():
    ctx = _lib.Context(0)
    text = b"ACGTTGCAACGTAGGCTA"
    starts = np.array([0, 6, 6, 12], dtype=np.uint32)
    g = DocumentSuffixTable([text[0:6], b"", text[6:12], text[12:]]).table()
    for metric, iupac, best, strands in MIXES:
        kf = _kf(1, metric, iupac, best, strands)
        tot, off, _, _ = _abi(ctx, text, g, [], kf, 0, starts)                  # nq = 0
        assert tot == 0 and off.tolist() == [0]
        for empty_starts in ([0], [0, 0, 0]):                                  # n = 0
            tot, off, pos, _ = _abi(ctx, b"", [], [b"AC", b"", b"G"], kf, 4, np.array(empty_starts, np.uint32))
            assert tot == 0 and off.tolist() == [0, 0, 0, 0] and (pos == MARK).all()
        a = _fetch(ctx, text, g, [b"ACG", b"GCA", b"T", b""], kf, starts)
        b = _fetch(ctx, text, g, [b"ACG", b"GCA", b"T", b""], kf, starts)
        assert _same(a, b) and int(a[0][-1]) > 0
    rng = np.random.default_rng(440)
    t = gen.dna(200_000)
    st = DocumentSuffixTable([_u8(t)[a:a + 1000] for a in range(0, 200_000, 1000)])
    qs = _reads(t, rng, 300, 40, 0.02, 0.01)
    for metric, k, best, strands in (("hamming", 3, None, "both"), ("edit", 2, None, "forward"),
                                     ("edit", 3, 0, "both")):
        a = st.approximate_documents_batch(qs, k, metric=metric, best=best, strands=strands)
        b = st.approximate_documents_batch(qs, k, metric=metric, best=best, strands=strands)
        assert _same(a, b) and int(a[0][-1]) > 0
    ctx.close()


@pytest.mark.parametrize("shift", [(1, 3), (3, 2)])
def test_unaligned_buffers(shift):
    rng = np.random.default_rng(450)
    text = _masked_dna(rng, 900) + bytes(range(256))
    qs = [bytes(b if b in b"ACGT" else 67 for b in text.upper()[a:a + m])
          for m in (1, 3, 9, 17) for a in rng.integers(0, 880, 5)] + [b"NNN", b"GAATTC"]
    ctx = _lib.Context(0)
    starts = np.array([0, 300, 300, 900], dtype=np.uint32)
    g, _ = ctx.docs_build(np.frombuffer(text, dtype=np.uint8), starts, with_lcp=False)
    docs = [text[0:300], b"", text[300:900], text[900:]]
    for metric, k, iupac, best, strands in (("hamming", 0, False, None, "forward"), ("hamming", 2, True, None, "both"),
                                            ("edit", 1, False, 0, "both"), ("edit", 2, True, 1, "forward")):
        kf = _kf(k, metric, iupac, best, strands)
        assert _same(_fetch(ctx, text, g, qs, kf, starts, shift=shift),
                     model_approx_docs.brute(docs, qs, k, metric, iupac, best, strands)), k
    ctx.close()


def test_bad_arguments():
    ctx = _lib.Context(0)
    text = b"ACGTACGTNNacgtGAATTC"
    sa = SuffixTable(text).table()
    starts = np.array([0, 8, 8], dtype=np.uint32)
    g = DocumentSuffixTable([text[:8], b"", text[8:]]).table()
    for extra in (0, EDIT, BEST | (1 << 8), IUPAC | BOTH, BEST | EDIT | IUPAC | BOTH):
        with pytest.raises(_lib.B200SAError) as e:                             # bit 29 on the single-text entry
            _abi(ctx, text, sa, [b"ACG"], 1 | extra | DOCS, 0)
        msg = str(e.value)
        assert e.value.code == BAD_ARG and "B200SA_APPROX_MAX_K" in msg and "DOCUMENTS" not in msg, hex(extra)
        for bit in (19, 22, 23, 26, 30):                                       # another unknown bit with the flag
            with pytest.raises(_lib.B200SAError) as e:
                _abi(ctx, text, g, [b"ACG"], 1 | extra | DOCS | (1 << bit), 0, starts)
            msg = str(e.value)
            assert e.value.code == BAD_ARG and "B200SA_APPROX_MAX_K" in msg and "B200SA_APPROX_DOCUMENTS" in msg, bit
    for bad in ([1, 5], [0, 7, 3], [0, 30]):
        with pytest.raises(_lib.B200SAError) as e:
            _abi(ctx, text, g, [b"ACG"], 1 | DOCS, 0, np.asarray(bad, np.uint32))
        assert e.value.code == BAD_ARG and "doc_starts rejected" in str(e.value)
    for off in ([1, 3], [0, 3, 2, 4], [0, 5, 3]):
        with pytest.raises(_lib.B200SAError) as e:
            _abi(ctx, text, g, [b"ACGT"], 1 | DOCS | BOTH, 0, starts, off=off)
        assert e.value.code == BAD_ARG and "q_off rejected" in str(e.value)
    with pytest.raises(_lib.B200SAError) as e:                                 # the IUPAC byte check, as without
        _abi(ctx, text, g, [b"ACGT", b"AC-G"], 1 | IUPAC | DOCS, 0, starts)
    assert e.value.code == BAD_ARG and "0x2d" in str(e.value) and "offset 6" in str(e.value)
    st = DocumentSuffixTable([text])
    for kw in (dict(metric="levenshtein"), dict(best=True), dict(iupac=1), dict(strands="reverse")):
        with pytest.raises(ValueError):
            st.approximate_documents(b"ACG", 1, **kw)
        with pytest.raises(ValueError):
            st.approximate_document_frequencies([b"ACG"], 1, **kw)
    with pytest.raises(ValueError):
        st.approximate_documents_batch([b"ACG"], 32)
    assert _same(_fetch(ctx, text, g, [b"ACG"], 1 | DOCS, starts),
                 model_approx_docs.brute([text[:8], b"", text[8:]], [b"ACG"], 1))
    ctx.close()
