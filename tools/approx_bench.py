"""f-14: approximate positions (b200sa_approx_positions_dev, b200sa_docs_approx_positions_dev) on device-resident
tables.  Prints one JSON line: card and power limit; per arm (the single text, and the same text cut into
documents of about 1 kB), workload and k the median CUDA-event time (one warm-up, then --reps) of the count
call plus the fetch call, the phase split of one timed fetch call, the candidates verified (the sizes of the
pieces' table ranges, from b200sa_positions_dev on the pieces), the occurrences found, and whether the first
--sample queries agree with tests/approx_check.c, whose time on one host core is reported beside them.

    python tools/approx_bench.py [--n 100000000] [--reps 5] [--sample 3]

Text: G_dna, as bench.py.  Workloads: 100 k reads of 150 bytes sampled from the text with 1 % substitutions, at
k = 0, 2, 4, 8 (pieces of 150 / (k + 1) bytes: few candidates beyond the read's own place); 1 k 20-mers sampled
from the text at k = 0..3, the shape of an off-target search, whose pieces are 5 bytes long at k = 3: about
n / 4^5 candidates per piece, the expensive regime."""
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
from tests import approx_check
from tools.docs_bench import card, cut, phase_times, timed

ALPHA = np.frombuffer(b"ACGT", dtype=np.uint8)


def mutate(a, rng, rate):
    sub = rng.random(a.shape) < rate
    a[sub] = rng.choice(ALPHA, int(sub.sum()))
    return a


def workloads(text, rng):
    n = len(text)
    at = rng.integers(0, n - 150, 100_000)
    reads = mutate(text[at[:, None] + np.arange(150)[None, :]].copy(), rng, 0.01)
    at20 = rng.integers(0, n - 20, 1000)
    mers = text[at20[:, None] + np.arange(20)[None, :]].copy()
    return [("reads_100k_x150_sub1pct", reads, (0, 2, 4, 8)), ("20mers_1k", mers, (0, 1, 2, 3))]


class Arm:
    """One device-resident table: the single text (starts None) or the documents."""

    def __init__(self, ctx, s, text, starts):
        self.ctx, self.s, self.text, self.starts = ctx, s, text, starts
        self.n = n = len(text)
        self.d_t = torch.from_numpy(text).cuda()
        self.d_sa = torch.empty(n, dtype=torch.int32, device="cuda")
        if starts is None:
            ctx.build_dev(self.d_t.data_ptr(), n, self.d_sa.data_ptr(), s)
        else:
            self.d_s = torch.from_numpy(starts.view(np.int32).copy()).cuda()
            ctx.docs_build_dev(self.d_t.data_ptr(), n, self.d_s.data_ptr(), len(starts), self.d_sa.data_ptr(), 0, s)
        torch.cuda.synchronize()

    def approx(self, d_q, d_off, nq, k, d_o, d_pos=0, d_mis=0, cap=0):
        if self.starts is None:
            return self.ctx.approx_positions_dev(self.d_t.data_ptr(), self.n, self.d_sa.data_ptr(), d_q, d_off, nq, k,
                                                 d_o, d_pos, d_mis, cap, self.s)
        return self.ctx.docs_approx_positions_dev(self.d_t.data_ptr(), self.n, self.d_sa.data_ptr(),
                                                  self.d_s.data_ptr(), len(self.starts), d_q, d_off, nq, k, d_o,
                                                  d_pos, d_mis, cap, self.s)

    def ranges(self, d_q, d_off, nq):
        d_s, d_e = torch.empty(nq, dtype=torch.int32, device="cuda"), torch.empty(nq, dtype=torch.int32, device="cuda")
        if self.starts is None:
            self.ctx.positions_dev(self.d_t.data_ptr(), self.n, self.d_sa.data_ptr(), d_q, d_off, nq, d_s.data_ptr(),
                                   d_e.data_ptr(), self.s)
        else:
            self.ctx.docs_positions_dev(self.d_t.data_ptr(), self.n, self.d_sa.data_ptr(), self.d_s.data_ptr(),
                                        len(self.starts), d_q, d_off, nq, d_s.data_ptr(), d_e.data_ptr(), self.s)
        torch.cuda.synchronize()
        return d_s.cpu().numpy().view(np.uint32).astype(np.int64), d_e.cpu().numpy().view(np.uint32).astype(np.int64)


def candidates(arm, reads, k):
    """The candidates the call verifies: the sizes of the table ranges of the k + 1 pieces of every query."""
    nq, m = reads.shape
    P = k + 1
    cuts = [j * m // P for j in range(P + 1)]
    pieces = np.concatenate([reads[:, cuts[j]:cuts[j + 1]] for j in range(P)], axis=1).reshape(-1)
    lens = np.tile(np.diff(cuts), nq)
    off = np.zeros(len(lens) + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    d_p, d_off = torch.from_numpy(pieces).cuda(), torch.from_numpy(off.view(np.int64)).cuda()
    s, e = arm.ranges(d_p.data_ptr(), d_off.data_ptr(), len(lens))
    return int((e - s).sum())


def run(arm, stream, reads, k, reps, sample):
    nq, m = reads.shape
    blob = reads.reshape(-1)
    off = (np.arange(nq + 1, dtype=np.uint64) * m)
    d_q = torch.from_numpy(blob).cuda()
    d_off = torch.from_numpy(off.view(np.int64)).cuda()
    d_o = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
    total = arm.approx(d_q.data_ptr(), d_off.data_ptr(), nq, k, d_o.data_ptr())
    pos = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")
    mis = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")

    def both():                                   # the protocol a caller follows: count, then fetch
        arm.approx(d_q.data_ptr(), d_off.data_ptr(), nq, k, d_o.data_ptr())
        arm.approx(d_q.data_ptr(), d_off.data_ptr(), nq, k, d_o.data_ptr(), pos.data_ptr(), mis.data_ptr(), total)

    both()
    ts = [timed(stream, both) for _ in range(reps)]
    arm.ctx.set_timing(True)
    arm.approx(d_q.data_ptr(), d_off.data_ptr(), nq, k, d_o.data_ptr(), pos.data_ptr(), mis.data_ptr(), total)
    phases = {p: round(v, 3) for p, v in phase_times(arm.ctx)}
    arm.ctx.set_timing(False)
    torch.cuda.synchronize()
    o = d_o.cpu().numpy().view(np.uint64)
    q1 = min(sample, nq)
    t0 = time.perf_counter()
    want = approx_check.approx_blob(arm.text, arm.starts, blob, off, k, 0, q1)
    base = time.perf_counter() - t0
    e = int(o[q1])
    agree = (np.array_equal(o[:q1 + 1], want[0]) and np.array_equal(pos[:e].cpu().numpy().view(np.uint32), want[1])
             and np.array_equal(mis[:e].cpu().numpy().view(np.uint32), want[2]))
    ms = statistics.median(ts)
    return {"k": k, "queries": nq, "query_len": m, "candidates": candidates(arm, reads, k), "occurrences": total,
            "count_plus_fetch_ms_median": round(ms, 3), "count_plus_fetch_ms_all": [round(x, 3) for x in ts],
            "queries_per_s": round(nq / ms * 1e3), "fetch_phases_ms": phases,
            "baseline_one_core": {"what": "tests/approx_check.c, a serial sliding window with early exit, one host core",
                                  "queries": q1, "s_per_query": round(base / max(q1, 1), 3)},
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
        for wname, reads, ks in work:
            res[wname] = [run(arm, stream, reads, k, a.reps, a.sample) for k in ks]
        out[arm_name] = res
        del arm
        torch.cuda.empty_cache()
    out["agree"] = all(r["agree"] for arm in ("text", "documents_1kB") for w, _, _ in work for r in out[arm][w])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
