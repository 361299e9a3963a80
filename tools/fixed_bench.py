"""f-21: fixed symbols in IUPAC queries (B200SA_APPROX_FIXED on b200sa_docs_approx_positions_dev, the text as one
document) on a device-resident table.  Prints one JSON line: card and power limit; per metric and k, with and
without the flag, the median CUDA-event time (one warm-up, then --reps) of the count call plus the fetch call and
the occurrences found.  For Hamming it also checks that the flagged list equals the unflagged list filtered on
the host to the windows whose PAM matches, and reports the time of that filter (numpy, host).

    python tools/fixed_bench.py [--n 100000000] [--reps 5]

Text: G_dna, as bench.py.  Workload, the off-target search of f-17 and f-18: 1 k random 20-nt guides, searched on
both strands at Hamming k = 3 and edit k = 2, each once as guide + "ngg" with the flag (the PAM fixed) and once as
guide + "NGG" without it (the PAM spends the threshold like the spacer)."""
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
from tools.approx_bench import Arm
from tools.docs_bench import card, timed

EDIT, IUPAC, FIXED, BOTH = 0x10000, 0x1000000, 0x2000000, 0x10000000
MINUS = 0x80000000


def run(arm, stream, qs, kf, reps):
    """(median ms, all ms, offsets, positions, distances) of count + fetch."""
    nq = len(qs)
    off = np.zeros(nq + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(q) for q in qs])
    d_q = torch.from_numpy(np.frombuffer(b"".join(qs), dtype=np.uint8).copy()).cuda()
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
    return (statistics.median(ts), ts, d_o.cpu().numpy().view(np.uint64),
            pos[:total].cpu().numpy().view(np.uint32), dist[:total].cpu().numpy().view(np.uint32))


def pam_filter(text, off, pos, dist):
    """The hits of guide + NGG whose GG holds: T[p + 21, p + 23) = GG on +, T[p, p + 2) = CC on -."""
    t = text
    p = pos.astype(np.int64)
    minus = (dist & np.uint32(MINUS)) != 0
    plus_ok = (t[np.minimum(p + 21, len(t) - 1)] == ord("G")) & (t[np.minimum(p + 22, len(t) - 1)] == ord("G"))
    minus_ok = (t[p] == ord("C")) & (t[np.minimum(p + 1, len(t) - 1)] == ord("C"))
    keep = np.where(minus, minus_ok, plus_ok)
    q = np.repeat(np.arange(len(off) - 1), np.diff(off.astype(np.int64)))
    o = np.zeros(len(off), dtype=np.uint64)
    o[1:] = np.cumsum(np.bincount(q[keep], minlength=len(off) - 1))
    return o, pos[keep], dist[keep]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    ctx = _lib.Context(0)
    text = gen.dna(a.n)
    rng = np.random.default_rng(1)
    spacers = [bytes(rng.choice(list(b"ACGT"), 20).tolist()) for _ in range(1000)]
    arm = Arm(ctx, stream.cuda_stream, text, np.zeros(1, dtype=np.uint32))
    out = {"gpu": name, "power_limit": power, "text": "G_dna", "n": a.n, "reps": a.reps, "guides": len(spacers),
           "strands": "both"}
    agree = True
    for metric, k in (("hamming", 3), ("edit", 2)):
        base = k | IUPAC | BOTH | (EDIT if metric == "edit" else 0)
        ms0, ts0, o0, p0, d0 = run(arm, stream, [s + b"NGG" for s in spacers], base, a.reps)
        ms1, ts1, o1, p1, d1 = run(arm, stream, [s + b"ngg" for s in spacers], base | FIXED, a.reps)
        r = {"without_flag": {"occurrences": int(o0[-1]), "count_plus_fetch_ms_median": round(ms0, 3),
                              "count_plus_fetch_ms_all": [round(x, 3) for x in ts0]},
             "with_flag": {"occurrences": int(o1[-1]), "count_plus_fetch_ms_median": round(ms1, 3),
                           "count_plus_fetch_ms_all": [round(x, 3) for x in ts1]}}
        if metric == "hamming":
            ts = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                f = pam_filter(text, o0, p0, d0)
                ts.append((time.perf_counter() - t0) * 1e3)
            same = all(np.array_equal(x, y) for x, y in zip(f, (o1, p1, d1)))
            r["host_filter"] = {"what": "the unflagged list filtered to intact PAMs with numpy, one host thread",
                                "ms_median": round(statistics.median(ts), 3), "equals_flagged": bool(same)}
            agree = agree and same
        out["%s_k%d" % (metric, k)] = r
    out["agree"] = bool(agree)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
