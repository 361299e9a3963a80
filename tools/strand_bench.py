"""f-18: approximate positions on both DNA strands (B200SA_APPROX_BOTH_STRANDS on b200sa_approx_positions_dev and
b200sa_docs_approx_positions_dev) on device-resident tables.  Prints one JSON line: card and power limit; per arm
(the single text, and the same text cut into documents of about 1 kB), workload, metric, k and best the median
CUDA-event time (one warm-up, then --reps) of the count call plus the fetch call with the flag, the same for the
composed way a caller has without it, whether the two agree bit for bit, the occurrences and minus-strand
occurrences, and whether the first --sample queries agree with the serial C statements run on q and rc(q) and
merged on the host, whose time on one host core is reported beside them.

    python tools/strand_bench.py [--n 100000000] [--reps 5] [--sample 1] [--arms text,documents_1kB]

Text: G_dna, as bench.py.  Workloads, the shapes of an off-target search and of read mapping: 1 k CRISPR guides
(20-mers sampled from the text with 5 % substitutions) + NGG under B200SA_APPROX_IUPAC at Hamming k = 0..4 and edit
k = 1, 2; 100 k reads of 150 bytes sampled from the text with 1 % substitutions (and 0.5 % insertions or deletions
for the edit arms), every second one reverse-complemented, at Hamming k = 4 and at edit k = 4 with and without
best=0.  The composed way is one call without the flag on queries + rc(queries), count then fetch, followed by a
device merge into one (p, strand) list per query: a torch sort of (query, p, strand) keys, and with best=0 a
per-query minimum over both strands and a filter before it, since separate queries would each get their own best."""
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
from tests import approx_check, edit_check, iupac_check, model_best, model_strand
from tools.approx_bench import Arm, mutate
from tools.docs_bench import card, cut, timed
from tools.edit_bench import reads_with_indels

EDIT, BEST, IUPAC, BOTH = 0x10000, 0x100000, 0x1000000, 0x10000000
MINUS = 0x80000000


def workloads(text, rng):
    n = len(text)
    at = rng.integers(0, n - 20, 1000)
    guides = mutate(text[at[:, None] + np.arange(20)[None, :]].copy(), rng, 0.05)
    guides = [g.tobytes() + b"NGG" for g in guides]
    at = rng.integers(0, n - 150, 100_000)
    sub = mutate(text[at[:, None] + np.arange(150)[None, :]].copy(), rng, 0.01)
    sub = [r.tobytes() for r in sub]
    ind = [r.tobytes() for r in reads_with_indels(text, rng, 100_000, 150, 0.01, 0.005)]
    flip = lambda rs: [model_strand.revcomp(r) if i % 2 else r for i, r in enumerate(rs)]
    return [("guides_1k_x20_NGG", guides, True,
             [("hamming", k, None) for k in range(5)] + [("edit", 1, None), ("edit", 2, None)]),
            ("reads_100k_x150_sub1pct_both_strands", flip(sub), False, [("hamming", 4, None)]),
            ("reads_100k_x150_sub1pct_indel05pct_both_strands", flip(ind), False, [("edit", 4, None), ("edit", 4, 0)])]


class Batch:
    """Queries on the device with their offsets and an offsets output."""

    def __init__(self, qs):
        self.nq = len(qs)
        self.blob = np.frombuffer(b"".join(qs), dtype=np.uint8).copy()
        self.off = np.zeros(self.nq + 1, dtype=np.uint64)
        self.off[1:] = np.cumsum([len(q) for q in qs])
        self.d_q = torch.from_numpy(self.blob).cuda()
        self.d_off = torch.from_numpy(self.off.view(np.int64)).cuda()
        self.d_o = torch.empty(self.nq + 1, dtype=torch.int64, device="cuda")

    def call(self, arm, kf, pos=None, dist=None, cap=0):
        return arm.approx(self.d_q.data_ptr(), self.d_off.data_ptr(), self.nq, kf, self.d_o.data_ptr(),
                          0 if pos is None else pos.data_ptr(), 0 if dist is None else dist.data_ptr(), cap)


def composed_merge(o2, pos, dist, nq, best):
    """The device merge of the composed way: the lists of entries 0..2nq (q, then rc(q) at nq + q) into one list
    per query by (p, strand), distances of minus hits with MINUS; best: cut both strands to d <= best(q) + best."""
    counts = (o2[1:] - o2[:-1])
    entry = torch.repeat_interleave(torch.arange(2 * nq, device="cuda"), counts)
    q, minus = entry % nq, entry >= nq
    p, d = pos.long() & 0xFFFFFFFF, dist.long() & 0xFFFFFFFF
    if best is not None:
        lo = torch.full((nq,), 1 << 40, dtype=torch.int64, device="cuda").scatter_reduce(0, q, d, "amin")
        keep = d <= lo[q] + best
        q, minus, p, d = q[keep], minus[keep], p[keep], d[keep]
    order = torch.argsort((q << 34) | (p << 1) | minus.long())
    off = torch.zeros(nq + 1, dtype=torch.int64, device="cuda")
    off[1:] = torch.cumsum(torch.bincount(q, minlength=nq), 0)
    v = (d | (minus.long() << 31))[order]
    return off, p[order].int(), torch.where(v >= 1 << 31, v - (1 << 32), v).int()


def c_statement(arm, qs, k, metric, iupac):
    """The serial C statements on q and rc(q), merged on the host: (offsets, pos, d | MINUS)."""
    out = []
    for q in qs:
        rc = model_strand.revcomp(q, iupac)
        if iupac:
            fw, rv = (iupac_check.iupac(arm.text, arm.starts, [x], k, metric) for x in (q, rc))
        else:
            check = approx_check.approx if metric == "hamming" else edit_check.edit
            fw, rv = (check(arm.text, arm.starts, [x], k) for x in (q, rc))
        out.append(model_strand.merge(model_best.lists(fw)[0], model_best.lists(rv)[0]))
    off = np.zeros(len(out) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(h) for h in out])
    return (off, np.asarray([p for h in out for p, _ in h], np.uint32),
            np.asarray([d for h in out for _, d in h], np.uint32))


def run(arm, stream, qs, both_batch, iupac, metric, k, best, reps, sample):
    nq = len(qs)
    one = Batch(qs)
    kf = k | (EDIT if metric == "edit" else 0) | (IUPAC if iupac else 0)
    kb = kf | BOTH | (0 if best is None else (best << 8) | BEST)
    total = one.call(arm, kb)
    pos = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")
    dist = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")

    def flag():                                   # the protocol a caller follows: count, then fetch
        one.call(arm, kb)
        one.call(arm, kb, pos, dist, total)

    total2 = both_batch.call(arm, kf)
    pos2 = torch.empty(max(total2, 1), dtype=torch.int32, device="cuda")
    dist2 = torch.empty(max(total2, 1), dtype=torch.int32, device="cuda")
    res = {}

    def composed():
        both_batch.call(arm, kf)
        both_batch.call(arm, kf, pos2, dist2, total2)
        res["out"] = composed_merge(both_batch.d_o, pos2[:total2], dist2[:total2], nq, best)

    flag()
    composed()
    tf = [timed(stream, flag) for _ in range(reps)]
    tc = [timed(stream, composed) for _ in range(reps)]
    torch.cuda.synchronize()
    o = one.d_o.cpu().numpy().view(np.uint64)
    got = (o, pos[:total].cpu().numpy().view(np.uint32), dist[:total].cpu().numpy().view(np.uint32))
    c_off, c_pos, c_dist = res["out"]
    same = (np.array_equal(got[0].astype(np.int64), c_off.cpu().numpy())
            and np.array_equal(got[1], c_pos.cpu().numpy().view(np.uint32))
            and np.array_equal(got[2], c_dist.cpu().numpy().view(np.uint32)))
    q1 = min(sample, nq)
    t0 = time.perf_counter()
    want = c_statement(arm, qs[:q1], k, metric, iupac)
    base = time.perf_counter() - t0
    e = int(o[q1])
    if best is not None:                          # best(q) over both strands, from the C statements' lists
        lists = model_best.lists(want)
        lists = [[h for h in hs if h[1] & (MINUS - 1) <= min(d & (MINUS - 1) for _, d in hs) + best] for hs in lists]
        want = (np.r_[0, np.cumsum([len(h) for h in lists])].astype(np.uint64),
                np.asarray([p for h in lists for p, _ in h], np.uint32),
                np.asarray([d for h in lists for _, d in h], np.uint32))
    agree = (np.array_equal(o[:q1 + 1], want[0]) and np.array_equal(got[1][:e], want[1])
             and np.array_equal(got[2][:e], want[2]))
    mf, mc = statistics.median(tf), statistics.median(tc)
    return {"metric": metric, "k": k, "best": best, "queries": nq, "occurrences": total,
            "minus_occurrences": int((got[2] >> 31).sum()),
            "flag_count_plus_fetch_ms_median": round(mf, 3), "flag_ms_all": [round(x, 3) for x in tf],
            "composed_ms_median": round(mc, 3), "composed_ms_all": [round(x, 3) for x in tc],
            "flag_over_composed": round(mf / mc, 3), "composed_agrees": bool(same),
            "baseline_one_core": {"what": "tests/approx_check.c, edit_check.c or iupac_check.c on q and rc(q), "
                                          "merged on the host, one host core", "queries": q1,
                                  "s_per_query": round(base / max(q1, 1), 3)},
            "agree": bool(agree)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=1)
    ap.add_argument("--arms", default="text,documents_1kB", help="comma-separated subset of the two tables")
    a = ap.parse_args()
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    s = stream.cuda_stream
    ctx = _lib.Context(0)
    text = gen.dna(a.n)
    work = workloads(text, np.random.default_rng(1))
    out = {"gpu": name, "power_limit": power, "text": "G_dna", "n": a.n, "reps": a.reps}
    names = a.arms.split(",")
    for arm_name, starts in (("text", None), ("documents_1kB", cut(a.n, 500, 1500, 1))):
        if arm_name not in names:
            continue
        arm = Arm(ctx, s, text, starts)
        res = {"docs": 1 if starts is None else len(starts)}
        for wname, qs, iupac, arms in work:
            both_batch = Batch(qs + [model_strand.revcomp(q, iupac) for q in qs])
            res[wname] = []
            for metric, k, best in arms:
                res[wname].append(run(arm, stream, qs, both_batch, iupac, metric, k, best, a.reps, a.sample))
                print(arm_name, wname, metric, k, best, res[wname][-1]["flag_count_plus_fetch_ms_median"],
                      file=sys.stderr, flush=True)          # progress, off the JSON line
            del both_batch
        out[arm_name] = res
        del arm
        torch.cuda.empty_cache()
    rows = [r for arm in names for w, _, _, _ in work for r in out[arm][w]]
    out["agree"] = all(r["agree"] for r in rows)
    out["composed_agrees"] = all(r["composed_agrees"] for r in rows)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
