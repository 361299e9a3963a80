"""f-17: approximate positions of queries in IUPAC nucleotide codes (B200SA_APPROX_IUPAC on
b200sa_approx_positions_dev and b200sa_docs_approx_positions_dev) on device-resident tables.  Prints one JSON
line: card and power limit; per arm (the single text, and the same text cut into documents of about 1 kB),
workload, metric and k the median CUDA-event time (one warm-up, then --reps) of the count call plus the fetch
call, the candidates verified (the sizes of the pieces' table ranges, from b200sa_positions_dev on the stretch
pieces of tests/model_iupac.py; n for a whole-table query), the occurrences found, and whether the first
--sample queries agree with tests/iupac_check.c, whose time on one host core is reported beside them.

    python tools/iupac_bench.py [--n 100000000] [--reps 5] [--sample 3]

Text: G_dna, as bench.py.  Workloads, the shapes of an off-target and a primer search: 1 k CRISPR guides (20-mers
sampled from the text with 5 % substitutions) + NGG at Hamming k = 0..4 and edit k = 1, 2; 1 k 20-mers sampled
from the text with three random two- or three-base codes at Hamming k = 0..3; one whole-table query, N x 21 + GG
at Hamming k = 3, which verifies every rank and shows the cost of the fallback."""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _lib, gen
from tests import iupac_check, model_iupac
from tools.approx_bench import Arm, mutate
from tools.docs_bench import card, cut, timed

IUPAC, EDIT = 0x1000000, 0x10000
FOLD = b"RYSWKMBDHV"


def workloads(text, rng):
    n = len(text)
    at = rng.integers(0, n - 20, 1000)
    guides = mutate(text[at[:, None] + np.arange(20)[None, :]].copy(), rng, 0.05)
    guides = [g.tobytes() + b"NGG" for g in guides]
    at = rng.integers(0, n - 20, 1000)
    mers = []
    for a in at:
        q = bytearray(text[a:a + 20].tobytes())
        for x in rng.choice(20, 3, replace=False):
            q[int(x)] = FOLD[int(rng.integers(0, len(FOLD)))]
        mers.append(bytes(q))
    return [("guides_1k_x20_NGG", guides, [("hamming", k) for k in range(5)] + [("edit", 1), ("edit", 2)]),
            ("degenerate_20mers_1k", mers, [("hamming", k) for k in range(4)]),
            ("whole_table_N21GG", [b"N" * 21 + b"GG"], [("hamming", 3)])]


def candidates(arm, qs, k):
    """The ranks the call verifies: per query the table ranges of its k + 1 stretch pieces, or n (whole table)."""
    pieces, whole = [], 0
    for q in qs:
        pcs = model_iupac.pieces(q, k)
        if pcs is None:
            whole += arm.n
        else:
            pieces += [q[o:o + L] for o, L in pcs]
    if not pieces:
        return whole
    off = np.zeros(len(pieces) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(p) for p in pieces])
    d_p = torch.from_numpy(np.frombuffer(b"".join(pieces), dtype=np.uint8).copy()).cuda()
    d_off = torch.from_numpy(off.view(np.int64)).cuda()
    s, e = arm.ranges(d_p.data_ptr(), d_off.data_ptr(), len(pieces))
    return whole + int((e - s).sum())


def run(arm, stream, qs, metric, k, reps, sample):
    nq = len(qs)
    blob = np.frombuffer(b"".join(qs), dtype=np.uint8).copy()
    off = np.zeros(nq + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(q) for q in qs])
    kf = k | IUPAC | (EDIT if metric == "edit" else 0)
    d_q = torch.from_numpy(blob).cuda()
    d_off = torch.from_numpy(off.view(np.int64)).cuda()
    d_o = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
    total = arm.approx(d_q.data_ptr(), d_off.data_ptr(), nq, kf, d_o.data_ptr())
    pos = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")
    dist = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")

    def both():                                   # the protocol a caller follows: count, then fetch
        arm.approx(d_q.data_ptr(), d_off.data_ptr(), nq, kf, d_o.data_ptr())
        arm.approx(d_q.data_ptr(), d_off.data_ptr(), nq, kf, d_o.data_ptr(), pos.data_ptr(), dist.data_ptr(), total)

    both()
    ts = [timed(stream, both) for _ in range(reps)]
    torch.cuda.synchronize()
    o = d_o.cpu().numpy().view(np.uint64)
    q1 = min(sample, nq)
    t0 = time.perf_counter()
    want = iupac_check.iupac_blob(arm.text, arm.starts, blob, off, k, metric, 0, q1)
    base = time.perf_counter() - t0
    e = int(o[q1])
    agree = (np.array_equal(o[:q1 + 1], want[0]) and np.array_equal(pos[:e].cpu().numpy().view(np.uint32), want[1])
             and np.array_equal(dist[:e].cpu().numpy().view(np.uint32), want[2]))
    ms = statistics.median(ts)
    return {"metric": metric, "k": k, "queries": nq, "candidates": candidates(arm, qs, k), "occurrences": total,
            "count_plus_fetch_ms_median": round(ms, 3), "count_plus_fetch_ms_all": [round(x, 3) for x in ts],
            "baseline_one_core": {"what": "tests/iupac_check.c, a serial class-count window or class-aware Sellers "
                                          "sweep, one host core", "queries": q1,
                                  "s_per_query": round(base / max(q1, 1), 3)},
            "agree": bool(agree)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=3)
    a = ap.parse_args()
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    s = stream.cuda_stream
    ctx = _lib.Context(0)
    text = gen.dna(a.n)
    work = workloads(text, np.random.default_rng(1))
    out = {"gpu": name, "power_limit": power, "text": "G_dna", "n": a.n, "reps": a.reps}
    for arm_name, starts in (("text", None), ("documents_1kB", cut(a.n, 500, 1500, 1))):
        arm = Arm(ctx, s, text, starts)
        res = {"docs": 1 if starts is None else len(starts)}
        for wname, qs, arms in work:
            res[wname] = [run(arm, stream, qs, metric, k, a.reps, a.sample) for metric, k in arms]
        out[arm_name] = res
        del arm
        torch.cuda.empty_cache()
    out["agree"] = all(r["agree"] for arm in ("text", "documents_1kB") for w, _, _ in work for r in out[arm][w])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
