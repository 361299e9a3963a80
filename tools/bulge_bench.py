"""f-22: separate budgets for mismatches, DNA bulges and RNA bulges (B200SA_APPROX_BULGES on
b200sa_docs_approx_positions_dev, the text as one document) on a device-resident table.  Prints one JSON line: card
and power limit, read in the same run; per budget (M, b_DNA, b_RNA), the median CUDA-event time (one warm-up, then
--reps) of the count call plus the fetch call, the occurrences found and the candidates the filter verifies, and
the same for the plain edit call at k = M + b_DNA + b_RNA on the same queries.

    python tools/bulge_bench.py [--n 100000000] [--reps 5] [--guides 1000]

Text: G_dna, as bench.py.  Workload, the CRISPR off-target search: 1 k random 20-nt guides + "ngg" with the PAM
fixed (B200SA_APPROX_IUPAC | B200SA_APPROX_FIXED), on both strands, at (4, 1, 1) and (3, 1, 0).  Candidates are the
ranks of the P = k + 1 pieces' table ranges over both strands (the IUPAC piece rule of include/b200sa.h), each
verified once per piece."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _lib, gen
from tools.approx_bench import Arm
from tools.docs_bench import card
from tools.fixed_bench import run

EDIT, BULGES, IUPAC, FIXED, BOTH = 0x10000, 0x200000, 0x1000000, 0x2000000, 0x10000000
COMP = bytes.maketrans(b"ACGTacgtNn", b"TGCAtgcaNn")


def pieces(q, P):
    """The pieces of IUPAC query q for P pieces, uppercased: the stretches of A C G T cut as b200sa.h states."""
    runs, x = [], 0
    while x < len(q):
        if q[x:x + 1].upper() in (b"A", b"C", b"G", b"T"):
            y = x
            while y < len(q) and q[y:y + 1].upper() in (b"A", b"C", b"G", b"T"):
                y += 1
            runs.append((x, y - x))
            x = y
        else:
            x += 1
    if sum(L for _, L in runs) < P:
        return None                                       # the whole-table slot
    t = max(t for t in range(1, len(q) + 1) if sum(L // t for _, L in runs) >= P)
    out = []
    for a, L in runs:
        c = min(L // t, P - len(out))
        out += [q[a + i * L // c:a + (i + 1) * L // c].upper() for i in range(c)]
    return out


def candidates(arm, qs, P):
    ps = []
    for q in qs:
        for s in (q, q.translate(COMP)[::-1]):
            got = pieces(s, P)
            if got is None:
                return None
            ps += got
    off = np.zeros(len(ps) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(p) for p in ps])
    d_q = torch.from_numpy(np.frombuffer(b"".join(ps), dtype=np.uint8).copy()).cuda()
    d_off = torch.from_numpy(off.view(np.int64)).cuda()
    s, e = arm.ranges(d_q.data_ptr(), d_off.data_ptr(), len(ps))
    return int((e.astype(np.int64) - s.astype(np.int64)).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--guides", type=int, default=1000)
    a = ap.parse_args()
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    ctx = _lib.Context(0)
    text = gen.dna(a.n)
    rng = np.random.default_rng(1)
    qs = [bytes(rng.choice(list(b"ACGT"), 20).tolist()) + b"ngg" for _ in range(a.guides)]
    arm = Arm(ctx, stream.cuda_stream, text, np.zeros(1, dtype=np.uint32))
    out = {"gpu": name, "power_limit": power, "text": "G_dna", "n": a.n, "reps": a.reps, "guides": len(qs),
           "query": "20-nt guide + ngg, PAM fixed", "strands": "both"}
    for m, d, r in ((4, 1, 1), (3, 1, 0)):
        k = m + d + r
        res = {}
        for what, kf in (("bulges", m | (d << 17) | (r << 22) | BULGES), ("edit", k)):
            ms, ts, off, _, _ = run(arm, stream, qs, kf | EDIT | IUPAC | FIXED | BOTH, a.reps)
            res[what] = {"occurrences": int(off[-1]), "count_plus_fetch_ms_median": round(ms, 3),
                         "count_plus_fetch_ms_all": [round(x, 3) for x in ts]}
        res["candidates"] = candidates(arm, qs, k + 1)
        res["pieces"] = k + 1
        out["M%d_dna%d_rna%d" % (m, d, r)] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
