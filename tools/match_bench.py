"""f-10: matching statistics and SMEMs (b200sa_match_stats_dev, b200sa_docs_match_stats_dev,
b200sa_smems_dev) on device-resident tables.  Prints one JSON line: card and power limit; per arm (the single
text, and the same text cut into documents of about 1 kB) and workload the median CUDA-event time (one
warm-up, then --reps) of the full call and of the lengths-only call, pattern positions/s and query bytes/s
(one pattern position per query byte), the phase split of one timed full call, and whether a sample of the
arrays equals the baseline's; SMEMs at min_len = 20 on the first workload (count call + fetch call), and on
the documents arm b200sa_docs_topk_dev (k = 10) over the SMEM ranges.

    python tools/match_bench.py [--n 100000000] [--reps 5]

Text: G_dna, as bench.py.  Workloads: 100 k reads of 150 bytes sampled from the text with 1 % substitutions
(long matches); 100 k random 150-mers (matches of about log4 n bytes: the search depth dominates); one query
of n/10 bytes that is a slice of the text with 1 % substitutions.  The baseline is tests/match_check.c, a
serial statement of the same arrays (a plain binary search per position, the range by two more), on ONE
host core over the first --sample positions of each workload: its rate is named `baseline_one_core`."""
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
from tests import match_check
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
    rnd = rng.choice(ALPHA, (100_000, 150))
    a = int(rng.integers(0, n - n // 10))
    even = np.arange(100_001, dtype=np.uint64) * 150
    return [("reads_100k_x150_sub1pct", reads.reshape(-1), even),
            ("random_100k_x150", rnd.reshape(-1), even),
            ("slice_n10_sub1pct", mutate(text[a:a + n // 10].copy(), rng, 0.01), np.array([0, n // 10], dtype=np.uint64))]


class Arm:
    """One device-resident table: the single text (starts None) or the documents."""

    def __init__(self, ctx, s, text, starts):
        self.ctx, self.s, self.text, self.starts = ctx, s, text, starts
        self.n = n = len(text)
        self.d_t = torch.from_numpy(text).cuda()
        self.d_sa = torch.empty(n, dtype=torch.int32, device="cuda")
        self.d_lcp = torch.empty(n, dtype=torch.int32, device="cuda")
        if starts is None:
            ctx.build_lcp_dev(self.d_t.data_ptr(), n, self.d_sa.data_ptr(), self.d_lcp.data_ptr(), s)
        else:
            self.d_s = torch.from_numpy(starts.view(np.int32).copy()).cuda()
            ctx.docs_build_dev(self.d_t.data_ptr(), n, self.d_s.data_ptr(), len(starts), self.d_sa.data_ptr(),
                               self.d_lcp.data_ptr(), s)
        torch.cuda.synchronize()
        self.sa = self.d_sa.cpu().numpy().view(np.uint32)

    def stats(self, d_q, d_off, nq, qb, d_len, d_start, d_end, with_lcp=True):
        lcp = self.d_lcp.data_ptr() if with_lcp else 0
        if self.starts is None:
            self.ctx.match_stats_dev(self.d_t.data_ptr(), self.n, self.d_sa.data_ptr(), lcp, d_q, d_off, nq, qb,
                                     d_len, d_start, d_end, self.s)
        else:
            self.ctx.docs_match_stats_dev(self.d_t.data_ptr(), self.n, self.d_sa.data_ptr(), lcp, self.d_s.data_ptr(),
                                          len(self.starts), d_q, d_off, nq, qb, d_len, d_start, d_end, self.s)


def run(arm, stream, blob, off, reps, sample):
    ctx = arm.ctx
    nq, qb = len(off) - 1, len(blob)
    d_q = torch.from_numpy(blob).cuda()
    d_off = torch.from_numpy(off.view(np.int64)).cuda()
    d_len, d_start, d_end, d_len2 = (torch.empty(qb, dtype=torch.int32, device="cuda") for _ in range(4))
    full = lambda: arm.stats(d_q.data_ptr(), d_off.data_ptr(), nq, qb, d_len.data_ptr(), d_start.data_ptr(),
                             d_end.data_ptr())
    lens = lambda: arm.stats(d_q.data_ptr(), d_off.data_ptr(), nq, qb, d_len2.data_ptr(), 0, 0, with_lcp=False)
    full()
    lens()
    tf, tl = [], []
    for _ in range(reps):
        tf.append(timed(stream, full))
        tl.append(timed(stream, lens))
    ctx.set_timing(True)
    full()
    phases = {p: round(ms, 3) for p, ms in phase_times(ctx)}
    ctx.set_timing(False)
    torch.cuda.synchronize()
    x1 = min(sample, qb)
    t0 = time.perf_counter()
    want = match_check.stats(arm.text, arm.starts, arm.sa, blob, off, 0, x1)
    base = time.perf_counter() - t0
    got = [t[:x1].cpu().numpy().view(np.uint32) for t in (d_len, d_start, d_end)]
    agree = all(np.array_equal(a, b) for a, b in zip(got, want)) and bool(torch.equal(d_len, d_len2))
    ms, ms_l = statistics.median(tf), statistics.median(tl)
    res = {"queries": nq, "positions": qb, "mean_len": round(float(d_len.float().mean()), 2),
           "full_ms_median": round(ms, 3), "full_ms_all": [round(x, 3) for x in tf],
           "lengths_only_ms_median": round(ms_l, 3), "lengths_only_ms_all": [round(x, 3) for x in tl],
           "positions_per_s": round(qb / ms * 1e3), "query_bytes_per_s": round(qb / ms * 1e3),
           "lengths_only_positions_per_s": round(qb / ms_l * 1e3), "phases_ms": phases,
           "baseline_one_core": {"what": "tests/match_check.c, a serial port of the same arrays, one host core",
                                 "positions": x1, "positions_per_s": round(x1 / base)},
           "agree": agree}
    return res, (d_q, d_off, d_len, d_start, d_end)


def smems(arm, stream, blob, off, dev, reps, min_len=20, k=10):
    ctx, s = arm.ctx, arm.s
    d_q, d_off, d_len, d_start, d_end = dev
    nq, qb = len(off) - 1, len(blob)
    d_so = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
    total = ctx.smems_dev(d_off.data_ptr(), nq, qb, d_len.data_ptr(), min_len, d_so.data_ptr(), 0, 0, s)
    qpos = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")

    def both():                                   # the protocol a caller follows: count, then fetch
        ctx.smems_dev(d_off.data_ptr(), nq, qb, d_len.data_ptr(), min_len, d_so.data_ptr(), 0, 0, s)
        ctx.smems_dev(d_off.data_ptr(), nq, qb, d_len.data_ptr(), min_len, d_so.data_ptr(), qpos.data_ptr(), total, s)

    both()
    ts = [timed(stream, both) for _ in range(reps)]
    ctx.set_timing(True)
    ctx.smems_dev(d_off.data_ptr(), nq, qb, d_len.data_ptr(), min_len, d_so.data_ptr(), qpos.data_ptr(), total, s)
    phases = {p: round(ms, 3) for p, ms in phase_times(ctx)}
    ctx.set_timing(False)
    # the rule on the host
    ln = d_len.cpu().numpy().view(np.uint32).astype(np.int64)
    first = np.zeros(qb, dtype=bool)
    first[off[:-1][off[:-1] < qb].astype(np.int64)] = True
    flag = (ln >= min_len) & (first | (np.r_[0, ln[:-1]] <= ln))
    x = np.nonzero(flag)[0]
    q_of = np.searchsorted(off, x, side="right") - 1
    agree = (total == len(x) and np.array_equal(qpos[:total].cpu().numpy(), x - off[q_of].astype(np.int64)) and
             np.array_equal(d_so.cpu().numpy(), np.searchsorted(x, off.astype(np.int64))))
    res = {"min_len": min_len, "smems": total, "count_plus_fetch_ms_median": round(statistics.median(ts), 3),
           "count_plus_fetch_ms_all": [round(v, 3) for v in ts], "fetch_phases_ms": phases, "agree": bool(agree)}
    if arm.starts is None:
        return res
    # retrieval on the SMEM ranges: top-k documents per SMEM, and the ranges against docs_positions_dev on the strings
    at = torch.from_numpy(x).cuda()
    r_s, r_e, r_l = d_start[at].contiguous(), d_end[at].contiguous(), d_len[at].long()
    byd = torch.empty(arm.n, dtype=torch.int32, device="cuda")
    prev = torch.empty(arm.n, dtype=torch.int32, device="cuda")
    ndocs = len(arm.starts)
    ctx.docs_list_index_dev(arm.n, arm.d_sa.data_ptr(), arm.d_s.data_ptr(), ndocs, byd.data_ptr(), prev.data_ptr(), s)
    count = torch.empty(total, dtype=torch.int32, device="cuda")
    docs = torch.empty(total * k, dtype=torch.int32, device="cuda")
    tf = torch.empty(total * k, dtype=torch.int32, device="cuda")
    topk = lambda: ctx.docs_topk_dev(arm.n, arm.d_sa.data_ptr(), arm.d_s.data_ptr(), ndocs, byd.data_ptr(),
                                     prev.data_ptr(), r_s.data_ptr(), r_e.data_ptr(), total, k, count.data_ptr(),
                                     docs.data_ptr(), tf.data_ptr(), s)
    topk()
    tt = [timed(stream, topk) for _ in range(reps)]
    s_off = torch.zeros(total + 1, dtype=torch.int64, device="cuda")
    s_off[1:] = torch.cumsum(r_l, 0)
    idx = torch.repeat_interleave(at - s_off[:-1], r_l) + torch.arange(int(s_off[-1]), device="cuda")
    strings = d_q[idx].contiguous()
    p_s, p_e = torch.empty_like(r_s), torch.empty_like(r_e)
    ctx.docs_positions_dev(arm.d_t.data_ptr(), arm.n, arm.d_sa.data_ptr(), arm.d_s.data_ptr(), ndocs,
                           strings.data_ptr(), s_off.data_ptr(), total, p_s.data_ptr(), p_e.data_ptr(), s)
    torch.cuda.synchronize()
    res["topk"] = {"k": k, "ranges": total, "rows": int(count.sum()), "ms_median": round(statistics.median(tt), 3),
                   "ms_all": [round(v, 3) for v in tt],
                   "agree": bool(torch.equal(p_s, r_s)) and bool(torch.equal(p_e, r_e)) and bool((count >= 1).all())}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=60_000)
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
        for k, (wname, blob, off) in enumerate(work):
            res[wname], dev = run(arm, stream, blob, off, a.reps, a.sample)
            if k == 0:
                res["smems_of_" + wname] = smems(arm, stream, blob, off, dev, a.reps)
            del dev
        out[arm_name] = res
        del arm
        torch.cuda.empty_cache()
    out["agree"] = all(v["agree"] for r in (out["text"], out["documents_1kB"]) for v in r.values()
                       if isinstance(v, dict)) and out["documents_1kB"]["smems_of_" + work[0][0]]["topk"]["agree"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
