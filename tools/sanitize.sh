#!/bin/bash
# compute-sanitizer on small builds: every path of round 2 (direct / robust LMS sort, the 2-bit bucket sort and its
# overflow, induce variants,
# fused classifier, sharded world-1 entry points, LCP paths, rows f, the suffix tree, the document suffix array)
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
for variant in ("", "1", "2", "3", "4", "5", "6:no_cascade", "6:cascade_4096", "6:classify_tma"):
    os.environ.pop("B200SA_NO_CASCADE", None); os.environ.pop("B200SA_CASCADE_MAX", None); os.environ.pop("B200SA_CLASSIFY_TMA", None)
    if variant:
        os.environ["B200SA_INDUCE"] = variant[0]
    if variant.endswith("no_cascade"): os.environ["B200SA_NO_CASCADE"] = "1"
    if variant.endswith("cascade_4096"): os.environ["B200SA_CASCADE_MAX"] = "4096"
    if variant.endswith("classify_tma"): os.environ["B200SA_CLASSIFY_TMA"] = "1"
    c2 = _lib.Context(0)
    for name, t in (cases if not variant else cases[:2] + cases[4:5] + cases[-1:]):
        sa, lcp = c2.build_lcp(t)
        want = oracle.sais(t)
        assert np.array_equal(sa, want), (variant, name)
        assert np.array_equal(lcp, oracle.lcp_kasai(t, want)), (variant, name)
    c2.close()
for k in ("B200SA_INDUCE", "B200SA_NO_CASCADE", "B200SA_CASCADE_MAX", "B200SA_CLASSIFY_TMA"):
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
    os.environ["B200SA_CLASSIFY_V1"] = "1"
    assert np.array_equal(ctx.build(t), want), name
    del os.environ["B200SA_CLASSIFY_V1"]
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
print("sanitize workload ok")
PY
for tool in memcheck racecheck; do
  timeout 2400 compute-sanitizer --tool $tool --error-exitcode 9 python /tmp/san.py > gpurun_out/san_$tool.log 2>&1
  echo "$tool exit $?"; tail -5 gpurun_out/san_$tool.log
done
