"""f-7: the generalized suffix tree with document counts (b200sa_docs_tree_dev) against the single-text
tree stage (b200sa_suffix_tree_dev) on the same bytes.  Prints one JSON line: card and power limit,
and per cut of the text the median CUDA-event times of both calls (one warm-up, then --reps each,
alternated), the node counts, the phase split of one timed docs-tree call, the device workspace of a
docs-tree call on a fresh context in bytes per text byte, and (on the ~1 kB cut) whether the serial
builder of tests/docs_tree_check.c gives the same eight arrays.

    python tools/docs_tree_bench.py [--n 100000000] [--reps 5] [--no-check]

G and glcp come from b200sa_docs_build_dev, SA and LCP of the concatenation from
b200sa_build_lcp_dev; all inputs and outputs stay on the device.  Cuts: G_dna into documents of about
1 kB (500..1499 bytes) and about 100 kB (50,000..149,999 bytes), and n/4 copies of "ACGT"."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _lib, gen
from tools.docs_bench import card, cut, phase_times, timed

FIELDS = _lib.DOCS_TREE_FIELDS


def run(ctx, stream, text, starts, reps, check):
    n = len(text)
    s = stream.cuda_stream
    d_t = torch.from_numpy(text).cuda()
    d_s = torch.from_numpy(starts.view(np.int32).copy()).cuda()
    d_g = torch.empty(n, dtype=torch.int32, device="cuda")
    d_gl = torch.empty(n, dtype=torch.int32, device="cuda")
    ctx.docs_build_dev(d_t.data_ptr(), n, d_s.data_ptr(), len(starts), d_g.data_ptr(), d_gl.data_ptr(), s)
    d_sa = torch.empty(n, dtype=torch.int32, device="cuda")
    d_lcp = torch.empty(n, dtype=torch.int32, device="cuda")
    ctx.build_lcp_dev(d_t.data_ptr(), n, d_sa.data_ptr(), d_lcp.data_ptr(), s)
    del d_t
    cap = 2 * n
    outs = [torch.empty(cap, dtype=torch.int32, device="cuda") for _ in FIELDS]
    ptrs = [o.data_ptr() for o in outs]
    nodes = {}

    def dtree(c=ctx):
        nodes["docs_tree"] = c.docs_tree_dev(n, d_g.data_ptr(), d_gl.data_ptr(), d_s.data_ptr(), len(starts), ptrs,
                                             cap, s)

    def stree():
        nodes["suffix_tree"] = ctx.suffix_tree_dev(n, d_sa.data_ptr(), d_lcp.data_ptr(), ptrs[:6], cap, s)

    dtree()
    stree()
    td, ts = [], []
    for _ in range(reps):                        # alternated, so both see the same card state
        td.append(timed(stream, dtree))
        ts.append(timed(stream, stree))
    ctx.set_timing(True)
    dtree()
    phases = {p: round(ms, 3) for p, ms in phase_times(ctx)}
    ctx.set_timing(False)
    fresh = _lib.Context(0)                      # workspace of one call on a fresh context
    dtree(fresh)
    torch.cuda.synchronize()
    ws = round(fresh.stats()["workspace_bytes"] / n, 1)
    fresh.close()
    N = nodes["docs_tree"]
    dc = outs[FIELDS.index("doc_count")][:N]
    res = {"n": n, "docs": len(starts), "docs_tree_nodes": N, "suffix_tree_nodes": nodes["suffix_tree"],
           "docs_tree_dev_ms_median": round(statistics.median(td), 3), "docs_tree_dev_ms_all": [round(x, 3) for x in td],
           "suffix_tree_dev_ms_median": round(statistics.median(ts), 3),
           "suffix_tree_dev_ms_all": [round(x, 3) for x in ts], "docs_tree_phases_ms": phases,
           "workspace_bytes_per_text_byte": ws, "root_doc_count": int(dc[0]),
           "nodes_in_all_docs": int((dc == int(dc[0])).sum())}
    if check:
        from tests import docs_tree_check
        dtree()
        torch.cuda.synchronize()
        got = {f: o[:N].cpu().numpy().view(np.uint32) for f, o in zip(FIELDS, outs)}
        want = docs_tree_check.tree(d_g.cpu().numpy().view(np.uint32), d_gl.cpu().numpy().view(np.uint32), starts)
        res["agree"] = all(np.array_equal(got[f], want[f]) for f in FIELDS)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-check", action="store_true")
    a = ap.parse_args()
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    ctx = _lib.Context(0)
    n = a.n - a.n % 4
    t = gen.dna(n)
    out = {"gpu": name, "power_limit": power, "text": "G_dna", "n": n}
    out["docs_1kB"] = run(ctx, stream, t, cut(n, 500, 1500, 1), a.reps, not a.no_check)
    out["docs_100kB"] = run(ctx, stream, t, cut(n, 50_000, 150_000, 2), a.reps, False)
    acgt = np.tile(np.frombuffer(b"ACGT", np.uint8), n // 4)
    out["acgt_copies"] = run(ctx, stream, acgt, np.arange(0, n, 4, dtype=np.uint32), a.reps, False)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
