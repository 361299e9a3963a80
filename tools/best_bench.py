"""f-16: best approximate hits (B200SA_APPROX_BEST on b200sa_approx_positions_dev and
b200sa_docs_approx_positions_dev) on device-resident tables.  Prints one JSON line: card and power limit; per arm
(the single text, and the same text cut into documents of about 1 kB), workload, metric and k the median CUDA-event
time (one warm-up, then --reps) of the count call plus the fetch call at slack 0, slack 1 and without the flag,
the rounds run and the live queries of every round, the occurrences, the phase split of one timed slack-0 fetch
(each phase name summed over the rounds and groups that repeat it, with its number of occurrences), and whether
--sample queries with a hit in the plain call and --sample without one agree with best(q) from the serial C
statements (tests/approx_check.c, tests/edit_check.c).

    python tools/best_bench.py [--n 100000000] [--reps 5] [--sample 3]

Text: G_dna, as bench.py.  Workloads: 100 k reads of 150 bytes with 1 % substitutions and 0.5 % insertions or
deletions (tools/edit_bench.py) at k = 4 and 8, where most reads stop after a few rounds; 1 k 20-mers drawn
uniformly over ACGT at k = 3, where every round runs (under the Hamming metric most of them have no hit within 3):
there the rounds can cost more than the plain call."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _lib, gen
from tests import approx_check, edit_check
from tools.approx_bench import Arm
from tools.docs_bench import card, cut, phase_times
from tools.edit_bench import measure, reads_with_indels

EDIT = 0x10000                                   # B200SA_APPROX_EDIT
BEST = 0x100000                                  # B200SA_APPROX_BEST
METRICS = {"hamming": 0, "edit": EDIT}
CHECK = {"hamming": approx_check.approx_blob, "edit": edit_check.edit_blob}


def workloads(text, rng):
    reads = reads_with_indels(text, rng, 100_000, 150, 0.01, 0.005)
    mers = rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), (1000, 20))
    return [("reads_100k_x150_sub1pct_indel05pct", reads, (4, 8)), ("random_20mers_1k", mers, (3,))]


def live_per_round(o, dist, k, s):
    """The live queries of every round the device runs, from the plain call's lists at k: q is live in round t
    while it has no occurrence within t - 1, or t <= best(q) + s."""
    nq = len(o) - 1
    cnt = np.diff(o.astype(np.int64))
    best = np.full(nq, 1 << 20, dtype=np.int64)
    hit = cnt > 0
    best[hit] = np.minimum.reduceat(dist.astype(np.int64), o[:-1][hit].astype(np.int64)) if hit.any() else []
    out = []
    for t in range(k + 1):
        live = int(((best >= t) | (t <= best + s)).sum())
        if not live:
            break
        out.append(live)
    return out


def phase_split(arm, d_q, d_off, nq, kf, pos, dist, total):
    """{phase: [ms summed over its occurrences, occurrences]} of one fetch call: the rounds and the emission
    groups repeat the search's phase names."""
    d_o = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
    arm.ctx.set_timing(True)
    arm.approx(d_q.data_ptr(), d_off.data_ptr(), nq, kf, d_o.data_ptr(), pos.data_ptr(), dist.data_ptr(), total)
    split = {}
    for p, v in phase_times(arm.ctx):
        ms, count = split.get(p, (0.0, 0))
        split[p] = (ms + v, count + 1)
    arm.ctx.set_timing(False)
    torch.cuda.synchronize()
    return {p: [round(ms, 3), count] for p, (ms, count) in split.items()}


def sample_queries(o, sample):
    """The first `sample` queries with an occurrence in the plain call's offsets o, and the first `sample` without."""
    hit = np.diff(o.astype(np.int64)) > 0
    return np.flatnonzero(hit)[:sample].tolist() + np.flatnonzero(~hit)[:sample].tolist()


def run(arm, stream, reads, metric, k, reps, sample):
    nq, m = reads.shape
    blob = reads.reshape(-1)
    off = np.arange(nq + 1, dtype=np.uint64) * m
    d_q = torch.from_numpy(blob).cuda()
    d_off = torch.from_numpy(off.view(np.int64)).cuda()
    kf = k | METRICS[metric]
    pts, ptotal, _, po, ppos, pdist = measure(arm, stream, d_q, d_off, nq, kf, reps)
    pdist = pdist[:ptotal].cpu().numpy().view(np.uint32)
    picked = sample_queries(po, sample)
    want = CHECK[metric](arm.text, arm.starts, reads[picked].reshape(-1), np.arange(len(picked) + 1, dtype=np.uint64) * m,
                         k)
    res = {"k": k, "queries": nq, "query_len": m, "checked_queries": picked,
           "checked_with_hit": int((np.diff(want[0].astype(np.int64)) > 0).sum()),
           "plain": {"occurrences": ptotal, "count_plus_fetch_ms_median": round(statistics.median(pts), 3)}}
    agree = True
    for s in (0, 1):
        ts, total, _, o, pos, dist = measure(arm, stream, d_q, d_off, nq, kf | (s << 8) | BEST, reps)
        rounds = arm.ctx.stats()["doubling_rounds"]
        live = live_per_round(po, pdist, k, s)
        if s == 0:
            phases = phase_split(arm, d_q, d_off, nq, kf | BEST, pos, dist, total)
        pos, dist = pos[:total].cpu().numpy().view(np.uint32), dist[:total].cpu().numpy().view(np.uint32)
        for i, q in enumerate(picked):               # the C statement's list at k, cut to d <= min(k, best + s)
            wp, wd = want[1][int(want[0][i]):int(want[0][i + 1])], want[2][int(want[0][i]):int(want[0][i + 1])]
            keep = wd <= (min(k, int(wd.min()) + s) if len(wd) else -1)
            a, b = int(o[q]), int(o[q + 1])
            agree &= bool(np.array_equal(pos[a:b], wp[keep]) and np.array_equal(dist[a:b], wd[keep]))
        agree &= rounds == len(live)
        ms = statistics.median(ts)
        res["slack_%d" % s] = {"occurrences": total, "count_plus_fetch_ms_median": round(ms, 3),
                               "count_plus_fetch_ms_all": [round(x, 3) for x in ts], "rounds": rounds,
                               "live_per_round": live, "vs_plain": round(ms / statistics.median(pts), 3)}
        if s == 0:
            res["slack_0"]["fetch_phases_ms"] = phases
    res["agree"] = bool(agree)
    print("%s k=%d n=%d: plain %.1f ms, slack 0 %.1f ms, agree %s" % (metric, k, nq, res["plain"]["count_plus_fetch_ms_median"],
          res["slack_0"]["count_plus_fetch_ms_median"], res["agree"]), file=sys.stderr, flush=True)
    return res


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
            res[wname] = {metric: [run(arm, stream, reads, metric, k, a.reps, a.sample) for k in ks]
                          for metric in METRICS}
        out[arm_name] = res
        del arm
        torch.cuda.empty_cache()
    out["agree"] = all(r["agree"] for arm in ("text", "documents_1kB") for w, _, _ in work for metric in METRICS
                       for r in out[arm][w][metric])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
