"""The alignments of approximate hits (B200SA_APPROX_ALIGN on b200sa_docs_approx_positions_dev, the
approximate_alignments* methods of SuffixTable and DocumentSuffixTable), for every mix of the edit metric, best
hits, IUPAC queries and both strands: bit for bit against tests/model_align.py on small collections, the hits
read back from the listing against approximate_positions_batch on large ones, the listing protocol, the limits
and the argument errors."""
import numpy as np
import pytest

from suffix_b200 import DocumentSuffixTable, SuffixTable, _approx, _lib, cigar_string, gen
from tests import model_align, model_docs, model_strand
from tests.test_gpu_approx import MARK, _abi, _fetch, _same
from tests.test_gpu_docs import _families, _u8
from tests.test_gpu_edit import _reads
from tests.test_gpu_iupac import _guides, _masked_dna
from tests.test_gpu_iupac import _queries as _iupac_queries
from tests.test_gpu_strand import _dna_queries

pytestmark = pytest.mark.gpu

BAD_ARG, TOO_LARGE = -1, -2
EDIT = 0x10000                                  # B200SA_APPROX_EDIT
BEST = 0x100000                                 # B200SA_APPROX_BEST
IUPAC = 0x1000000                               # B200SA_APPROX_IUPAC
BOTH = 0x10000000                               # B200SA_APPROX_BOTH_STRANDS
DOCS = 0x20000000                               # B200SA_APPROX_DOCUMENTS
ALIGN = 0x8000000                               # B200SA_APPROX_ALIGN
MINUS = model_strand.MINUS
METRIC = {"hamming": 0, "edit": EDIT}
MIXES = [(metric, iupac, best, strands) for metric in ("hamming", "edit") for iupac in (False, True)
         for best in (None, 0, 1) for strands in ("forward", "both")]


def _kf(k, metric, iupac, best, strands, align=True):
    return (k | METRIC[metric] | (IUPAC if iupac else 0) | (0 if best is None else (best << 8) | BEST) |
            (BOTH if strands == "both" else 0) | (ALIGN if align else 0))


def _with_minus(res, strands):
    """(offsets, positions, distances | MINUS, ends, cigar_offsets, cigar) of what the batch method returns."""
    if strands == "forward":
        return res
    off, pos, dist, minus, ends, coff, cig = res
    assert minus.dtype == bool and not (dist & MINUS).any()
    return off, pos, dist | np.where(minus, np.uint32(MINUS), np.uint32(0)), ends, coff, cig


def _positions(st, qs, k, kw):
    res = st.approximate_positions_batch(qs, k, **kw)
    if kw["strands"] == "forward":
        return res
    off, pos, dist, minus = res
    return off, pos, dist | np.where(minus, np.uint32(MINUS), np.uint32(0))


def _check_hits(st, qs, k, kw, got):
    """The hits read back from the listing are approximate_positions_batch's, and each hit's words obey the
    stated properties (vectorised over the listing)."""
    off, pos, dist, ends, coff, cig = _with_minus(got, kw["strands"])
    assert _same((off, pos, dist), _positions(st, qs, k, kw))
    m = np.array([len(q) for q in qs], dtype=np.int64)[np.repeat(np.arange(len(qs)), np.diff(off.astype(np.int64)))]
    h = len(pos)
    assert coff.dtype == np.uint64 and len(coff) == h + 1 and cig.dtype == np.uint32 and not (cig & MINUS).any()
    if h == 0:
        return
    hit = np.repeat(np.arange(h), np.diff(coff.astype(np.int64)))
    lens, code = (cig >> 4).astype(np.int64), cig & 15
    assert np.isin(code, [1, 2, 7, 8]).all() and (lens > 0).all()
    span = lambda codes: np.bincount(hit, np.where(np.isin(code, codes), lens, 0), minlength=h).astype(np.int64)
    assert np.array_equal(span([8, 1, 2]), dist & (MINUS - 1))
    assert np.array_equal(span([7, 8, 1]), m)
    assert np.array_equal(span([7, 8, 2]), ends.astype(np.int64) - pos)
    last = coff[1:].astype(np.int64) - 1
    assert (code[last] != 2).all() and (np.diff(coff.astype(np.int64)) <= 2 * (dist & (MINUS - 1)) + 1).all()
    starts = np.asarray(st.doc_starts() if hasattr(st, "doc_starts") else [0], dtype=np.int64)
    doc_end = np.append(starts[1:], len(st))[np.searchsorted(starts, pos, side="right") - 1]
    assert (ends <= doc_end).all()
    if kw["metric"] == "hamming":
        assert (ends.astype(np.int64) == pos + m).all()


@pytest.mark.parametrize("metric,iupac,best,strands", MIXES)
def test_families_equal_model(metric, iupac, best, strands):
    rng = np.random.default_rng(600 + MIXES.index((metric, iupac, best, strands)))
    sets = _families(rng)[::8] + [[_masked_dna(rng, int(rng.integers(1, 100))) for _ in range(3)] for _ in range(6)]
    sets += [[b"", _masked_dna(rng, 60), b"", b"ACGT"]]                      # empty documents, a short last one
    ctx = _lib.Context(0)
    kw = dict(metric=metric, iupac=iupac, best=best, strands=strands)
    for i, docs in enumerate(sets):
        k = [0, 1, 2, 3, 4][i % 5]
        if iupac:
            qs = _iupac_queries(rng, docs, k)
        else:
            qs = _dna_queries(rng, docs, k) + [b"\x01z", b"TTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTT"]
        g, _ = model_docs.brute(docs)
        text, starts = model_docs.concat(docs)
        want = model_align.listing(docs, qs, k, metric, iupac, best, strands)
        assert _same(_fetch(ctx, text, g, qs, _kf(k, metric, iupac, best, strands), starts), want), (docs, k)
        st = DocumentSuffixTable(docs)
        got = st.approximate_alignments_batch(qs, k, **kw)
        hoff, pos, dist, minus, ends, coff, cig = _approx._hits(*want)
        assert _same(_with_minus(got, strands),
                     (hoff, pos, dist | np.where(minus, np.uint32(MINUS), np.uint32(0)), ends, coff, cig)), (docs, k)
        _check_hits(st, qs, k, kw, got)
        one = st.approximate_alignments(qs[-1], k, **kw)
        assert _same(one, st.approximate_alignments_batch([qs[-1]], k, **kw)[1:])
        if len(docs) == 1:                                         # a single text through the documents entry
            assert _same(SuffixTable(text).approximate_alignments_batch(qs, k, **kw), got), (docs, k)
    ctx.close()


def test_single_text_equals_one_document():
    rng = np.random.default_rng(610)
    text = _masked_dna(rng, 5000).upper()
    qs = _reads(np.frombuffer(text, dtype=np.uint8), rng, 200, 30, 0.03, 0.02) + [b"", b"GAATTC", b"AC"]
    t1, d1 = SuffixTable(text), DocumentSuffixTable([text])
    for metric, k, best, strands in (("hamming", 2, None, "both"), ("edit", 3, None, "forward"),
                                     ("edit", 2, 0, "both"), ("edit", 4, 1, "both")):
        kw = dict(metric=metric, best=best, strands=strands)
        a, b = t1.approximate_alignments_batch(qs, k, **kw), d1.approximate_alignments_batch(qs, k, **kw)
        assert _same(a, b) and int(a[0][-1]) > 0
        _check_hits(t1, qs, k, dict(kw, iupac=False), a)


@pytest.fixture(scope="module")
def large():
    """10^6 bases as one text and in ~1 kB documents, with reads (half reverse-complemented) and guides + NGG."""
    rng = np.random.default_rng(620)
    t = gen.dna(1_000_000)
    text = _u8(t)
    cuts = np.unique(rng.integers(1, len(t), 1000))
    kb = DocumentSuffixTable([text[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(t)])])
    reads = _reads(t, rng, 2000, 150, 0.01, 0.005)
    reads = [model_strand.revcomp(r) if i % 2 else r for i, r in enumerate(reads)]
    guides = [g for g in _guides(t, rng, 300) if g.endswith(b"NGG")]
    return [("text", SuffixTable(text), reads, guides), ("kb_documents", kb, reads, guides)]


@pytest.mark.parametrize("metric,iupac,best,strands", MIXES)
def test_large_hits_equal_approximate_positions(large, metric, iupac, best, strands):
    kw = dict(metric=metric, iupac=iupac, best=best, strands=strands)
    rng = np.random.default_rng(630)
    for name, st, reads, guides in large:
        qs, k = (guides, 3 if metric == "hamming" else 2) if iupac else (reads, 4 if metric == "hamming" else 3)
        got = st.approximate_alignments_batch(qs, k, **kw)
        _check_hits(st, qs, k, kw, got)
        off, pos, dist, ends, coff, cig = _with_minus(got, strands)
        assert int(off[-1]) > 0, name
        text = st.text()
        starts = np.asarray(st.doc_starts() if hasattr(st, "doc_starts") else [0], dtype=np.int64)
        q_of = np.repeat(np.arange(len(qs)), np.diff(off.astype(np.int64)))
        for i in rng.choice(len(pos), min(len(pos), 60), replace=False).tolist():   # a sample against the model
            p, d = int(pos[i]), int(dist[i])
            E = int(np.append(starts[1:], len(text))[np.searchsorted(starts, p, side="right") - 1])
            ops, end = model_align.align(text, E, p, qs[q_of[i]], d & (MINUS - 1), metric, iupac, d >= MINUS, True)
            assert model_align.words(ops) == cig[int(coff[i]):int(coff[i + 1])].tolist() and end == ends[i], (name, i)


def test_cap_protocol():
    rng = np.random.default_rng(640)
    text = _masked_dna(rng, 2000)
    starts = np.array([0, 300, 300, 1000, 1013], dtype=np.uint32)
    docs = [text[a:b] for a, b in zip(starts, list(starts[1:]) + [len(text)])]
    g = DocumentSuffixTable(docs).table()
    up = text.upper()
    qs = [bytes(b if b in b"ACGT" else 65 for b in up[a:a + 12]) for a in rng.integers(0, 1985, 12)]
    qs = qs + [model_strand.revcomp(q) for q in qs[:3]] + [b"GAATTC", b"", b"AN", b"AC"]
    ctx = _lib.Context(0)
    for metric, iupac, best, strands in MIXES[::2]:
        kf = _kf(2, metric, iupac, best, strands)
        want = model_align.listing(docs, qs, 2, metric, iupac, best, strands)
        total = int(want[0][-1])
        assert total > 1
        for cap in (0, 1, total - 1):                                        # offsets and total only
            tot, off, pos, dist = _abi(ctx, text, g, qs, kf, cap, starts, buf=total + 5)
            assert tot == total and np.array_equal(off, want[0])
            assert (pos == MARK).all() and (dist == MARK).all(), cap
        tot, off, pos, dist = _abi(ctx, text, g, qs, kf, total, starts, buf=total + 5)   # fits: nothing past total
        assert tot == total and np.array_equal(off, want[0])
        assert np.array_equal(pos[:total], want[1]) and np.array_equal(dist[:total], want[2])
        assert (pos[total:] == MARK).all() and (dist[total:] == MARK).all()
    ctx.close()


def test_edge_cases():
    ctx = _lib.Context(0)
    text = b"ACGTTGCAACGTAGGCTA"
    starts = np.array([0, 6, 6, 12], dtype=np.uint32)
    docs = [text[0:6], b"", text[6:12], text[12:]]
    g = DocumentSuffixTable(docs).table()
    for metric, iupac, best, strands in MIXES:
        kf = _kf(1, metric, iupac, best, strands)
        tot, off, _, _ = _abi(ctx, text, g, [], kf, 0, starts)                  # nq = 0
        assert tot == 0 and off.tolist() == [0]
        tot, off, pos, _ = _abi(ctx, b"", [], [b"AC", b"", b"G"], kf, 4, np.array([0], np.uint32))   # n = 0
        assert tot == 0 and off.tolist() == [0, 0, 0, 0] and (pos == MARK).all()
        qs = [b"ACG", b"GCA", b"T", b"", b"GGGGGGGGGG", b"CGTAGG", b"GCTA", b"TTGCAA", b"ACGT"]
        a = _fetch(ctx, text, g, qs, kf, starts)
        assert _same(a, model_align.listing(docs, qs, 1, metric, iupac, best, strands))
        assert _same(a, _fetch(ctx, text, g, qs, kf, starts))                   # repeated calls
    st = DocumentSuffixTable(docs)
    pos, dist, minus, ends, coff, cig = st.approximate_alignments(b"ACGT", 0, strands="both")   # a palindrome
    assert pos.tolist() == [0, 0, 8, 8] and minus.tolist() == [False, True] * 2 and not dist.any()
    assert ends.tolist() == [4, 4, 12, 12] and [cigar_string(cig[a:b]) for a, b in zip(coff[:-1], coff[1:])] == ["4="] * 4
    ctx.close()


def test_bad_arguments_and_limits():
    ctx = _lib.Context(0)
    text = b"ACGTACGTNNacgtGAATTC"
    sa = SuffixTable(text).table()
    starts = np.array([0, 8, 8], dtype=np.uint32)
    docs = [text[:8], b"", text[8:]]
    g = DocumentSuffixTable(docs).table()
    for extra in (0, EDIT, BEST | (1 << 8), IUPAC | BOTH, BEST | EDIT | IUPAC | BOTH):
        with pytest.raises(_lib.B200SAError) as e:                             # bit 27 on the single-text entry
            _abi(ctx, text, sa, [b"ACG"], 1 | extra | ALIGN, 0)
        assert e.value.code == BAD_ARG and "B200SA_APPROX_MAX_K" in str(e.value)
        assert "DOCUMENTS" not in str(e.value) and "ALIGN" not in str(e.value), hex(extra)
        with pytest.raises(_lib.B200SAError) as e:                             # with B200SA_APPROX_DOCUMENTS
            _abi(ctx, text, g, [b"ACG"], 1 | extra | ALIGN | DOCS, 0, starts)
        msg = str(e.value)
        assert e.value.code == BAD_ARG and "B200SA_APPROX_ALIGN" in msg and "B200SA_APPROX_DOCUMENTS" in msg
        with pytest.raises(_lib.B200SAError) as e:                             # NULL d_mismatches with cap > 0
            _abi(ctx, text, g, [b"ACG"], 1 | extra | ALIGN, 4, starts, with_mis=False)
        assert e.value.code == BAD_ARG and "d_mismatches" in str(e.value)
        for bit in (19, 22, 23, 26, 30):                                       # an unknown bit names both flags
            with pytest.raises(_lib.B200SAError) as e:
                _abi(ctx, text, g, [b"ACG"], 1 | extra | ALIGN | (1 << bit), 0, starts)
            msg = str(e.value)
            assert e.value.code == BAD_ARG and "B200SA_APPROX_DOCUMENTS" in msg and "B200SA_APPROX_ALIGN" in msg
        assert _same(_fetch(ctx, text, g, [b"ACG"], 1 | ALIGN, starts), model_align.listing(docs, [b"ACG"], 1))
    # the edit traceback takes queries up to B200SA_APPROX_ALIGN_MAX_M = 4096 bytes
    big = _u8(gen.dna(20_000))
    gb = DocumentSuffixTable([big]).table()
    sb = np.array([0], np.uint32)
    q = bytearray(big[5000:9096])
    q[100] = ord("A") if q[100] != ord("A") else ord("C")
    tot, off, _, _ = _abi(ctx, big, gb, [bytes(q)], 2 | EDIT | ALIGN, 0, sb)
    assert tot > 0
    assert _same(_fetch(ctx, big, gb, [bytes(q)], 2 | EDIT | ALIGN, sb),
                 model_align.listing([big], [bytes(q)], 2, "edit"))
    with pytest.raises(_lib.B200SAError) as e:
        _abi(ctx, big, gb, [bytes(q) + b"A"], 2 | EDIT | ALIGN, 0, sb)
    assert e.value.code == TOO_LARGE and "B200SA_APPROX_ALIGN_MAX_M" in str(e.value)
    tot, _, _, _ = _abi(ctx, big, gb, [big[5000:10000]], 2 | ALIGN, 0, sb)    # Hamming has no such limit
    assert tot == 1
    assert _same(_fetch(ctx, text, g, [b"ACG"], 1 | EDIT | ALIGN, starts),
                 model_align.listing(docs, [b"ACG"], 1, "edit"))               # the context stays usable
    st = DocumentSuffixTable([text])
    for kw in (dict(metric="levenshtein"), dict(best=True), dict(iupac=1), dict(strands="reverse")):
        with pytest.raises(ValueError):
            st.approximate_alignments(b"ACG", 1, **kw)
        with pytest.raises(ValueError):
            SuffixTable(text).approximate_alignments_batch([b"ACG"], 1, **kw)
    ctx.close()
