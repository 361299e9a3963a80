"""f-15: approximate positions within k edits (B200SA_APPROX_EDIT on b200sa_approx_positions_dev and
b200sa_docs_approx_positions_dev) on device-resident tables.  Prints one JSON line: card and power limit; per arm
(the single text, and the same text cut into documents of about 1 kB), workload and k the median CUDA-event
time (one warm-up, then --reps) of the count call plus the fetch call, the phase split of one timed fetch call,
the candidates verified (the sizes of the pieces' table ranges), the occurrences found, the same for the Hamming
call on the same queries, and whether the first --sample queries agree with tests/edit_check.c, whose time on
one host core is reported beside them.

    python tools/edit_bench.py [--n 100000000] [--reps 5] [--sample 3]

Text: G_dna, as bench.py.  Workloads: 100 k reads of 150 bytes sampled from the text with 1 % substitutions and
0.5 % insertions or deletions, at k = 0, 2, 4, 8; 1 k 20-mers sampled from the text at k = 0..3, whose pieces
are 5 bytes long at k = 3: about n / 4^5 candidates per piece, the expensive regime."""
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
from tests import edit_check
from tools.approx_bench import Arm, candidates
from tools.docs_bench import card, cut, phase_times, timed

EDIT = 0x10000                                   # B200SA_APPROX_EDIT
ALPHA = np.frombuffer(b"ACGT", dtype=np.uint8)


def reads_with_indels(text, rng, count, m, sub, indel):
    """count reads of m bytes sampled from the text with substitutions at rate sub and insertions or deletions
    at rate indel; a read that came out shorter is filled from the text that follows it, a longer one cut."""
    n = len(text)
    at = rng.integers(0, n - 2 * m, count)
    out = np.empty((count, m), dtype=np.uint8)
    for r, a in enumerate(at.tolist()):
        src = text[a:a + 2 * m].copy()
        w = src[:m].copy()
        s = rng.random(m) < sub
        w[s] = rng.choice(ALPHA, int(s.sum()))
        ev = np.flatnonzero(rng.random(m) < indel)
        if len(ev):
            w = list(w)
            for x in sorted(ev.tolist(), reverse=True):
                if rng.random() < 0.5:
                    del w[x]
                else:
                    w.insert(x, int(rng.choice(ALPHA)))
            w = np.asarray(w, dtype=np.uint8)
            if len(w) < m:
                w = np.concatenate([w, src[m:m + m - len(w)]])
        out[r] = w[:m]
    return out


def workloads(text, rng):
    reads = reads_with_indels(text, rng, 100_000, 150, 0.01, 0.005)
    at20 = rng.integers(0, len(text) - 20, 1000)
    mers = text[at20[:, None] + np.arange(20)[None, :]].copy()
    return [("reads_100k_x150_sub1pct_indel05pct", reads, (0, 2, 4, 8)), ("20mers_1k", mers, (0, 1, 2, 3))]


def measure(arm, stream, d_q, d_off, nq, k, reps):
    """(count + fetch times, occurrences, phases of one fetch, offsets, positions, distances) of one metric."""
    d_o = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
    total = arm.approx(d_q.data_ptr(), d_off.data_ptr(), nq, k, d_o.data_ptr())
    pos = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")
    dist = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")

    def both():                                   # the protocol a caller follows: count, then fetch
        arm.approx(d_q.data_ptr(), d_off.data_ptr(), nq, k, d_o.data_ptr())
        arm.approx(d_q.data_ptr(), d_off.data_ptr(), nq, k, d_o.data_ptr(), pos.data_ptr(), dist.data_ptr(), total)

    both()
    ts = [timed(stream, both) for _ in range(reps)]
    arm.ctx.set_timing(True)
    arm.approx(d_q.data_ptr(), d_off.data_ptr(), nq, k, d_o.data_ptr(), pos.data_ptr(), dist.data_ptr(), total)
    phases = {p: round(v, 3) for p, v in phase_times(arm.ctx)}
    arm.ctx.set_timing(False)
    torch.cuda.synchronize()
    return ts, total, phases, d_o.cpu().numpy().view(np.uint64), pos, dist


def run(arm, stream, reads, k, reps, sample):
    nq, m = reads.shape
    blob = reads.reshape(-1)
    off = (np.arange(nq + 1, dtype=np.uint64) * m)
    d_q = torch.from_numpy(blob).cuda()
    d_off = torch.from_numpy(off.view(np.int64)).cuda()
    ts, total, phases, o, pos, dist = measure(arm, stream, d_q, d_off, nq, k | EDIT, reps)
    hts, htotal, _, _, _, _ = measure(arm, stream, d_q, d_off, nq, k, reps)
    q1 = min(sample, nq)
    t0 = time.perf_counter()
    want = edit_check.edit_blob(arm.text, arm.starts, blob, off, k, 0, q1)
    base = time.perf_counter() - t0
    e = int(o[q1])
    agree = (np.array_equal(o[:q1 + 1], want[0]) and np.array_equal(pos[:e].cpu().numpy().view(np.uint32), want[1])
             and np.array_equal(dist[:e].cpu().numpy().view(np.uint32), want[2]))
    ms, hms = statistics.median(ts), statistics.median(hts)
    return {"k": k, "queries": nq, "query_len": m, "candidates": candidates(arm, reads, k), "occurrences": total,
            "count_plus_fetch_ms_median": round(ms, 3), "count_plus_fetch_ms_all": [round(x, 3) for x in ts],
            "queries_per_s": round(nq / ms * 1e3), "fetch_phases_ms": phases,
            "hamming": {"occurrences": htotal, "count_plus_fetch_ms_median": round(hms, 3)},
            "baseline_one_core": {"what": "tests/edit_check.c, a serial Sellers sweep with Ukkonen's cut-off, "
                                          "one host core", "queries": q1, "s_per_query": round(base / max(q1, 1), 3)},
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
