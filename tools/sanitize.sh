#!/bin/bash
# compute-sanitizer on small builds: every path of round 2 (direct / robust LMS sort, the 2-bit bucket sort and its
# overflow, both induce kernels with and without cascade steps,
# fused byte and packed classifiers, sharded world-1 entry points, LCP paths, rows f, the suffix tree, the document suffix array,
# the local-sort overflow, the direct path's probe and 64-bit round-0 keys)
mkdir -p gpurun_out
cat > /tmp/san.py <<'PY'
import sys, os
sys.path.insert(0, os.getcwd())
import numpy as np
import torch
from suffix_b200 import _lib, gen, sharded, SuffixTable, GeneralizedSuffixTable
from oracle import oracle
ctx = _lib.Context(0)
cases = [("dna", gen.dna(300_000)), ("dna_nl", gen.dna(200_001, newline_tail=True)), ("bytes", gen.rand_bytes(200_000)),
         ("english", gen.english(150_000)),
         ("runs", np.concatenate([gen.dna(5000), np.full(20000, 78, np.uint8), gen.dna(5000), np.full(300, 65, np.uint8)])),
         ("periodic", np.tile(np.frombuffer(b"abcab", np.uint8), 20000)),
         ("tiled", gen.tiled(gen.fixture("AP009048_10000.fasta"), 120_000))]
rng = np.random.default_rng(3)
runs = []
for k in range(300):
    runs.append(np.full(int(rng.integers(1, 12)), b"ACGT"[k % 4], dtype=np.uint8))
    runs.append(gen.dna(int(rng.integers(1, 40)), seed=k))
cases.append(("short_runs", np.concatenate(runs * 8)))
# 2-bit text with one top-16 bucket of > 4096 LMS suffixes: k_lms_bucket_sort overflows, the four-pass sort reruns
fill = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, (4200, 6))]
cases.append(("bucket_overflow", np.concatenate([gen.dna(20000)] + [np.concatenate([np.frombuffer(b"TACGTACGTC", np.uint8), f]) for f in fill] + [gen.dna(20000)])))
for variant in ("", "1", "6:no_cascade", "6:cascade_4096"):
    os.environ.pop("B200SA_NO_CASCADE", None); os.environ.pop("B200SA_CASCADE_MAX", None)
    if variant:
        os.environ["B200SA_INDUCE"] = variant[0]
    if variant.endswith("no_cascade"): os.environ["B200SA_NO_CASCADE"] = "1"
    if variant.endswith("cascade_4096"): os.environ["B200SA_CASCADE_MAX"] = "4096"
    c2 = _lib.Context(0)
    for name, t in (cases if not variant else cases[:2] + cases[4:5] + cases[-1:]):
        sa, lcp = c2.build_lcp(t)
        want = oracle.sais(t)
        assert np.array_equal(sa, want), (variant, name)
        assert np.array_equal(lcp, oracle.lcp_kasai(t, want)), (variant, name)
    c2.close()
for k in ("B200SA_INDUCE", "B200SA_NO_CASCADE", "B200SA_CASCADE_MAX"):
    os.environ.pop(k, None)
os.environ["B200SA_LMS_SORT4"] = "1"            # the four-pass LMS sort on 2-bit text
for name, t in cases[:1] + cases[-1:]:
    assert np.array_equal(ctx.build(t), oracle.sais(t)), name
del os.environ["B200SA_LMS_SORT4"]
from suffix_b200 import SuffixTree
sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
import tree_oracle
for name, t in cases + [("banana", np.frombuffer(b"banana", np.uint8)), ("a3000", np.full(3000, 97, np.uint8))]:
    tb = t.tobytes()
    st_t = SuffixTree(tb)
    want = oracle.sais(tb)
    ref = tree_oracle.suffix_tree(want, oracle.lcp_kasai(tb, want))
    assert all(np.array_equal(st_t.arrays()[f], ref[f]) for f in tree_oracle.FIELDS), name
for name, t in cases[:4]:
    want = oracle.sais(t)
    os.environ["B200SA_LCP_LINEAR"] = "1"
    assert np.array_equal(ctx.lcp(t, want), oracle.lcp_kasai(t, want)), name
    del os.environ["B200SA_LCP_LINEAR"]
    os.environ["B200SA_NO_DIRECT"] = "1"
    assert np.array_equal(ctx.build(t), want), name
    del os.environ["B200SA_NO_DIRECT"]
    d_t = torch.from_numpy(t.copy()).cuda()
    g, nm, st = sharded.lms_sort_sharded(ctx, d_t)
    d_sa = torch.from_numpy(want.astype(np.int64)).cuda().to(torch.int32)
    d_lcp = torch.empty(len(t), dtype=torch.int32, device="cuda")
    ctx.lcp_sharded(d_t.data_ptr(), len(t), d_sa.data_ptr(), d_lcp.data_ptr(), False, 0)
    torch.cuda.synchronize()
    assert np.array_equal(d_lcp.cpu().numpy().view(np.uint32), oracle.lcp_kasai(t, want)), name
st_ = SuffixTable(cases[0][1].tobytes())
st_.lcp_intervals()
g = GeneralizedSuffixTable([b"ACGT" * 50, b"GATTACA" * 30, b"TTTT"])
assert len(g.positions(b"TACAG")) > 0
from suffix_b200 import DocumentSuffixTable
from tests import model_docs
dna = gen.dna(60_000).tobytes()
doc_sets = [[dna[:20000], b"", dna[20000:20007], dna[:20000], dna[20000:]], [b"ACGT"] * 3000,
            [bytes(range(256)), b"\x00\x00", b"", bytes(range(256))[:7]], [b"banana"]]
for k, docs in enumerate(doc_sets):
    for two in ("", "1"):                        # the (lo, r, d) sort and the two-stage sort
        os.environ["B200SA_DOCS_SORT2"] = two
        dt = DocumentSuffixTable(docs)
        if len(dt) < 3000:
            g, l = model_docs.brute(docs)
            assert np.array_equal(dt.table(), g) and np.array_equal(dt.lcp_lens(), l), k
    s_, e_ = dt.positions_batch([b"ACG", b"TA", b"\x00", b"", b"GTAC"])
    assert all(int(a) <= int(b) for a, b in zip(s_, e_)), k
del os.environ["B200SA_DOCS_SORT2"]
from suffix_b200 import DocumentSuffixTree      # the generalized suffix tree and its document counts
for k, docs in enumerate(doc_sets + [[b"ACGT"] * 2000 + [b""]]):
    dtr = DocumentSuffixTree(docs)
    assert dtr.root().doc_count() == sum(1 for d in docs if d), k
    assert len(dtr.document_counts([b"ACG", b"TA", b"\x00", b"", b"GTAC"])) == 5, k
for k, docs in enumerate(doc_sets + [[b"ACGT"] * 2000 + [b""]]):   # document listing: index, listing, tf on / off
    dl = DocumentSuffixTable(docs)
    qs = [b"ACG", b"TA", b"\x00", b"", b"GTAC", b"A"]
    off, dd, tf = dl.documents_batch(qs, _cap_guess=1)             # cap too small, then sufficient
    assert np.array_equal(dl.documents_batch(qs)[1], dd), k
    assert np.array_equal(dl.document_frequencies(qs), np.diff(off.astype(np.int64))), k
    d_off, d_docs, _ = dl._list_dev(qs, max(1, int(off[-1])), with_tf=False)
    assert int(d_off[-1]) == int(off[-1]), k
# top-k: every size class (b"A" of 9000 copies: two levels of tiles), k = 1 / B200SA_TOPK_MAX, one and many rounds
for k, docs in enumerate(doc_sets + [[b"ACGT"] * 9000 + [b""]]):
    dl = DocumentSuffixTable(docs)
    qs = [b"ACG", b"TA", b"\x00", b"", b"GTAC", b"A", b"C"]
    for kk in (1, 1024):
        want = dl.top_documents_batch(qs, kk)
        os.environ["B200SA_TOPK_ROUND"] = "50"
        got = dl.top_documents_batch(qs, kk)
        del os.environ["B200SA_TOPK_ROUND"]
        assert all(np.array_equal(x, y) for x, y in zip(want, got)), (k, kk)
# matching statistics: both entry points, lengths only, SMEMs with cap too small then sufficient
ms_qs = [dna[100:180], dna[:40] + b"N" + dna[41:90], b"", b"\x00\x01", b"banana" * 3, bytes(range(256))]
single = SuffixTable(dna)
for k, tab in enumerate([single] + [DocumentSuffixTable(docs) for docs in doc_sets]):
    off, ln, s_, e_ = tab.matching_statistics(ms_qs)
    assert all(int(a) <= int(b) for a, b in zip(s_, e_)), k
    so, qpos, sl, _, _ = tab.smems(ms_qs, 2)                       # count call (cap = 0), then the fetch
    assert len(qpos) == int(so[-1]) and (sl >= 2).all(), k
blob = torch.from_numpy(np.frombuffer(b"".join(ms_qs), dtype=np.uint8).copy()).cuda()
d_qo = torch.from_numpy(np.cumsum([0] + [len(q) for q in ms_qs]).astype(np.int64)).cuda()
d_ln = torch.empty(len(blob), dtype=torch.int32, device="cuda")
d_t_, d_sa_, _ = single._device_arrays()
ctx.match_stats_dev(d_t_.data_ptr(), len(dna), d_sa_.data_ptr(), 0, blob.data_ptr(), d_qo.data_ptr(), len(ms_qs),
                    len(blob), d_ln.data_ptr(), 0, 0, 0)                          # lengths only, no lcp
torch.cuda.synchronize()
assert np.array_equal(d_ln.cpu().numpy().view(np.uint32), single.matching_statistics(ms_qs)[1])
# repeats: the three entry points, every mode, count call (cap = 0) then the fetch
for k, tab in enumerate([single] + [DocumentSuffixTable(docs) for docs in doc_sets]):
    assert len(tab.repeat_lengths()) == len(tab), k
    for L in (1, 4, 12):
        rs, re_, rf, rl_ = tab.repeated_substrings(L, with_ends=True)
        assert (re_ - rs >= 2).all() and (rf <= rl_).all(), (k, L)
        for mode in tab._REPEAT_MODES:
            sp = tab.duplicate_spans(L, mode)
            width = (sp[1] - sp[0]) if isinstance(sp, tuple) else (sp[:, 2] - sp[:, 1])
            assert int(width.astype(np.int64).sum()) == tab.duplicated_bytes(L, mode), (k, L, mode)
# LZ77: lpf, the count call (cap = 0) then the fetch, on the single text and every document set
for k, tab in enumerate([single] + [DocumentSuffixTable(docs) for docs in doc_sets]):
    lpf, src = tab.longest_previous_factors()
    fs, fl, fq = tab.lz77_factors()
    assert len(fs) == tab.lz77_count() and int(fl.astype(np.int64).sum()) == len(tab), k
# BWT: the forward (with r) and the inverse on the single text and every document set, at the default ruler
# spacing and at forced ones (every row a ruler, one in three, the terminator rows alone)
from suffix_b200 import inverse_bwt_documents
for k, tab in enumerate([single] + [DocumentSuffixTable(docs) for docs in doc_sets]):
    b, t = tab.bwt()
    assert tab.bwt_runs() >= 1, k
    for sp in (None, 1, 3, len(tab) + 1):
        if sp: os.environ["B200SA_BWT_RULER"] = str(sp)
        assert b"".join(inverse_bwt_documents(b, t)) == tab.text(), (k, sp)
        os.environ.pop("B200SA_BWT_RULER", None)
# approximate positions: the count call (cap = 0) then the fetch, on the single text, every document set, a
# repetitive text whose slots span many chunks, and queries of m <= k on documents with empty ones
ap_qs = [dna[a:a + 25] for a in range(0, 4000, 97)] + [b"", b"A", b"ACG", b"ACGTACGT"]
for k, tab in enumerate([single] + [DocumentSuffixTable(docs) for docs in doc_sets] +
                        [SuffixTable(b"a" * 5000), DocumentSuffixTable([b"", b"ab", b"", b"c"])]):
    for kk in (0, 3, 31):
        off, pos, mis = tab.approximate_positions_batch(ap_qs + [b"a" * 9], kk)
        assert len(pos) == int(off[-1]) and (mis <= kk).all(), (k, kk)
# approximate positions within k edits: the same tables and queries with the edit metric, whose windows reach k
# past both sides of every candidate and whose band reaches 2k past them, near document ends included
for k, tab in enumerate([single] + [DocumentSuffixTable(docs) for docs in doc_sets] +
                        [SuffixTable(b"a" * 5000), DocumentSuffixTable([b"", b"ab", b"", b"c"])]):
    for kk in (0, 3, 31):
        off, pos, dist = tab.approximate_positions_batch(ap_qs + [b"a" * 9, b"A" * 40], kk, metric="edit")
        assert len(pos) == int(off[-1]) and (dist <= kk).all(), (k, kk)
# best hits: the same tables and queries in rounds over compacted batches (every query live, some, none), with
# one emission and scatter per final threshold, for both metrics
for k, tab in enumerate([single] + [DocumentSuffixTable(docs) for docs in doc_sets] +
                        [SuffixTable(b"a" * 5000), DocumentSuffixTable([b"", b"ab", b"", b"c"])]):
    for kk, sl in ((0, 0), (3, 0), (3, 1), (31, 2)):
        for metric in ("hamming", "edit"):
            off, pos, dist = tab.approximate_positions_batch(ap_qs + [b"a" * 9, b"A" * 40], kk, metric=metric, best=sl)
            assert len(pos) == int(off[-1]) and (dist <= kk).all(), (k, kk, sl, metric)
# IUPAC queries: the canonical copy, the stretch pieces (a whole-table query among them) and the piece table read
# by both verifications, with and without best hits
iu_qs = [q[:20] + b"NGG" for q in ap_qs if len(q) >= 20] + [b"N" * 21 + b"GG", b"RYACGTNNacgu", b"", b"n"]
for k, tab in enumerate([single] + [DocumentSuffixTable(docs) for docs in doc_sets] +
                        [SuffixTable(b"A" * 5000), DocumentSuffixTable([b"", b"AC", b"", b"G"])]):
    for kk, sl in ((0, None), (3, None), (31, None), (3, 1)):
        for metric in ("hamming", "edit"):
            off, pos, dist = tab.approximate_positions_batch(iu_qs, kk, metric=metric, best=sl, iupac=True)
            assert len(pos) == int(off[-1]) and (dist <= kk).all(), (k, kk, sl, metric)
# both strands: the doubled batch (plain and canonical complements), the key merge and, with best hits, the pair
# rounds, the staging scatter and the staged merge
for k, tab in enumerate([single] + [DocumentSuffixTable(docs) for docs in doc_sets] +
                        [SuffixTable(b"A" * 5000), DocumentSuffixTable([b"", b"AC", b"", b"G"])]):
    for kk, sl in ((0, None), (3, None), (31, None), (3, 0), (3, 1)):
        for metric in ("hamming", "edit"):
            for iu, qs in ((False, ap_qs + [b"GAATTC", b"a" * 9]), (True, iu_qs)):
                off, pos, dist, minus = tab.approximate_positions_batch(qs, kk, metric=metric, best=sl, iupac=iu,
                                                                        strands="both")
                assert len(pos) == len(minus) == int(off[-1]) and (dist <= kk).all(), (k, kk, sl, metric, iu)
# approximate document listing: the staged hit lists of every mix (one strand and both, plain and IUPAC, with and
# without best hits), the marks, their scan, the offsets, the emission and the least-distance pass, and the count
# call alone
for k, docs in enumerate(doc_sets + [[b"", b"AC", b"", b"G"], [b"A"] * 50 + [b""]]):
    tab = DocumentSuffixTable(docs)
    for kk, sl in ((0, None), (3, None), (31, None), (3, 0), (3, 1)):
        for metric in ("hamming", "edit"):
            for iu, qs in ((False, ap_qs + [b"GAATTC", b"a" * 9]), (True, iu_qs)):
                for strands in ("forward", "both"):
                    kw = dict(metric=metric, best=sl, iupac=iu, strands=strands)
                    res = tab.approximate_documents_batch(qs, kk, **kw)
                    off, ds, dist = res[:3]
                    assert len(ds) == int(off[-1]) and (dist <= kk).all() and (ds < len(docs)).all(), (k, kk, sl)
                    assert (tab.approximate_document_frequencies(qs, kk, **kw) == np.diff(off.astype(np.int64))).all()
# alignments of the hits: the staged hit lists of every mix, the Hamming and edit count kernels (one warp per hit,
# its move choices in shared memory), the scan, the offsets and the emission, and the count call alone; a single
# text goes through the documents entry
for k, docs in enumerate(doc_sets + [[b"", b"AC", b"", b"G"], [b"A"] * 50 + [b""]]):
    for tab in (DocumentSuffixTable(docs),) + ((SuffixTable(docs[0]),) if len(docs) == 1 else ()):
        for kk, sl in ((0, None), (3, None), (31, None), (3, 0), (3, 1)):
            for metric in ("hamming", "edit"):
                for iu, qs in ((False, ap_qs + [b"GAATTC", b"a" * 9]), (True, iu_qs)):
                    for strands in ("forward", "both"):
                        res = tab.approximate_alignments_batch(qs, kk, metric=metric, best=sl, iupac=iu,
                                                               strands=strands)
                        off, pos, dist = res[:3]
                        assert len(pos) == int(off[-1]) and (dist <= kk).all() and res[-2][-1] == len(res[-1]), k
# refinement branches (tests/test_gpu_refine.py): a local-sort overflow in round 2 of the direct path, the direct
# path's probe (2^20 tied after round 1, large groups), 64-bit round-0 keys of the reduced string
import ctypes
from tests.test_gpu_refine import motif_copies, probe_text
from tests.model_u32_sa import u32_sa
for name, t in (("local_overflow", motif_copies("bytes", 1026, seed=1026)), ("probe", probe_text(150, 7000, seed=150))):
    assert np.array_equal(ctx.build(t), oracle.sais(t)), name
R = np.random.default_rng(1).integers(0, 1 << 16, 1 << 20, dtype=np.uint32)
R[0] = (1 << 16) - 1                             # names = 2^16: 17-bit symbols, two of them per 64-bit key
out = np.empty(len(R), dtype=np.uint32)
rc = _lib.lib().b200sa_test_reduced_sa(ctx._h, R.ctypes.data, len(R), 1 << 16, out.ctypes.data, ctypes.byref(ctypes.c_uint32()))
assert rc == 0 and np.array_equal(out, u32_sa(R)), "reduced_sa 64-bit"
print("sanitize workload ok")
PY
for tool in memcheck racecheck; do
  timeout 2400 compute-sanitizer --tool $tool --error-exitcode 9 python /tmp/san.py > gpurun_out/san_$tool.log 2>&1
  echo "$tool exit $?"; tail -5 gpurun_out/san_$tool.log
done
