"""f-19: the documents that contain each query within k (B200SA_APPROX_DOCUMENTS on
b200sa_docs_approx_positions_dev) on device-resident document tables.  Prints one JSON line: card and power limit;
per workload the median CUDA-event time (one warm-up, then --reps) of the count call plus the fetch call for three
arms that compute the same listing, whether they agree bit for bit, and the numbers of hits and listed documents.

    python tools/approx_docs_bench.py [--reps 5] [--workloads pangenome,documents_1kB]

Arms: (a) the flag; (b) the composed way a caller has without it: approximate positions (count, fetch), the hits
copied to the host, each position's document found as locate() finds it (the last start <= p) and a per-query
unique-and-minimum on the host; (c) the same composition kept on the device with torch: searchsorted over the
document starts, unique_consecutive over (query, document) keys -- the hits are ordered by p within a query, so no
sort is needed -- and a segment minimum of (d << 1) | minus by scatter_reduce.

Workloads: a pangenome-shaped collection, 1,000 copies of one 100 kB G_dna genome (100 MB), each with seeded 1 %
substitutions and 0.1 % single-base insertions or deletions, searched with 1 k 20-nt guides + NGG from the base
genome under B200SA_APPROX_IUPAC on both strands at Hamming k = 3 and edit k = 2, and with 10 k 22-nt primers from
the base genome at Hamming k = 2 on both strands; and, for continuity with rows f-14 .. f-18, 100 MB G_dna cut into
~1 kB documents with 100 k reads of 150 bytes (1 % substitutions, 0.5 % insertions or deletions) at edit k = 4 with
best=0."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _lib, gen
from tools.approx_bench import ALPHA, Arm, mutate
from tools.docs_bench import card, cut, timed
from tools.edit_bench import reads_with_indels

EDIT, BEST, IUPAC, BOTH, DOCS = 0x10000, 0x100000, 0x1000000, 0x10000000, 0x20000000
MINUS = 0x80000000


def copies(base, count, rng, sub, indel):
    """The concatenation of count mutated copies of base and their starts."""
    out = []
    for _ in range(count):
        c = mutate(base.copy(), rng, sub)
        at = np.flatnonzero(rng.random(len(c)) < indel)
        ins = rng.random(len(at)) < 0.5
        c = np.insert(c, at[ins], rng.choice(ALPHA, int(ins.sum())))
        out.append(np.delete(c, at[~ins] + np.searchsorted(at[ins], at[~ins], side="right")))
    starts = np.r_[0, np.cumsum([len(c) for c in out[:-1]])].astype(np.uint32)
    return np.concatenate(out), starts


def samples(text, rng, count, m):
    at = rng.integers(0, len(text) - m, count)
    return text[at[:, None] + np.arange(m)[None, :]]


class Batch:
    """Queries on the device with their offsets and an offsets output."""

    def __init__(self, qs):
        self.nq = len(qs)
        blob = np.frombuffer(b"".join(qs), dtype=np.uint8).copy()
        off = np.zeros(self.nq + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(q) for q in qs])
        self.d_q = torch.from_numpy(blob).cuda()
        self.d_off = torch.from_numpy(off.view(np.int64)).cuda()
        self.d_o = torch.empty(self.nq + 1, dtype=torch.int64, device="cuda")

    def call(self, arm, kf, pos=None, dist=None, cap=0):
        return arm.approx(self.d_q.data_ptr(), self.d_off.data_ptr(), self.nq, kf, self.d_o.data_ptr(),
                          0 if pos is None else pos.data_ptr(), 0 if dist is None else dist.data_ptr(), cap)


def host_group(off, pos, dist, starts):
    """(b): per query the distinct documents of its hits and the least (d << 1) | minus in each, on the host."""
    nq = len(off) - 1
    q = np.repeat(np.arange(nq, dtype=np.int64), np.diff(off.astype(np.int64)))
    d = np.searchsorted(starts, pos, side="right").astype(np.int64) - 1
    w = ((dist & np.uint32(MINUS - 1)).astype(np.int64) << 1) | (dist >> 31).astype(np.int64)
    key = (q << 32) | d
    uniq, inv = np.unique(key, return_inverse=True)
    least = np.full(len(uniq), 1 << 40, dtype=np.int64)
    np.minimum.at(least, inv, w)
    o = np.zeros(nq + 1, dtype=np.uint64)
    o[1:] = np.cumsum(np.bincount(uniq >> 32, minlength=nq))
    return o, (uniq & 0xFFFFFFFF).astype(np.uint32), ((least >> 1) | ((least & 1) << 31)).astype(np.uint32)


def device_group(d_o, pos, dist, d_starts, nq):
    """(c): the same on the device with torch; the hits of a query are ordered by p, so (q, doc) keys come in runs."""
    q = torch.repeat_interleave(torch.arange(nq, device="cuda"), d_o.diff())
    p = pos.long() & 0xFFFFFFFF
    d = torch.searchsorted(d_starts, p, right=True) - 1
    dl = dist.long() & 0xFFFFFFFF
    w = ((dl & (MINUS - 1)) << 1) | (dl >> 31)
    key, inv = torch.unique_consecutive((q << 32) | d, return_inverse=True)
    least = torch.full((len(key),), 1 << 40, dtype=torch.int64, device="cuda").scatter_reduce(0, inv, w, "amin")
    o = torch.zeros(nq + 1, dtype=torch.int64, device="cuda")
    o[1:] = torch.cumsum(torch.bincount(key >> 32, minlength=nq), 0)
    return o, key & 0xFFFFFFFF, (least >> 1) | ((least & 1) << 31)


def run(arm, stream, qs, kf, reps):
    one = Batch(qs)
    nq = len(qs)
    kd = kf | DOCS
    ndocs = one.call(arm, kd)
    docs = torch.empty(max(ndocs, 1), dtype=torch.int32, device="cuda")
    dd = torch.empty(max(ndocs, 1), dtype=torch.int32, device="cuda")
    hits = one.call(arm, kf)
    pos = torch.empty(max(hits, 1), dtype=torch.int32, device="cuda")
    dist = torch.empty(max(hits, 1), dtype=torch.int32, device="cuda")
    d_starts = torch.from_numpy(arm.starts.astype(np.int64)).cuda()
    res = {}

    def flag():                                   # (a) the protocol a caller follows: count, then fetch
        one.call(arm, kd)
        one.call(arm, kd, docs, dd, ndocs)
        res["a"] = (one.d_o.cpu().numpy().view(np.uint64).copy(), docs[:ndocs].cpu().numpy().view(np.uint32),
                    dd[:ndocs].cpu().numpy().view(np.uint32))

    def host():                                   # (b) positions, then locate and group on the host
        one.call(arm, kf)
        one.call(arm, kf, pos, dist, hits)
        off = one.d_o.cpu().numpy().view(np.uint64)
        res["b"] = host_group(off, pos[:hits].cpu().numpy().view(np.uint32),
                              dist[:hits].cpu().numpy().view(np.uint32), arm.starts)

    def device():                                 # (c) positions, then the same composition with torch
        one.call(arm, kf)
        one.call(arm, kf, pos, dist, hits)
        o, dc, w = device_group(one.d_o, pos[:hits], dist[:hits], d_starts, nq)
        res["c"] = (o.cpu().numpy().astype(np.uint64), dc.cpu().numpy().astype(np.uint32),
                    w.cpu().numpy().astype(np.uint32))

    times = {}
    for name, fn in (("a_flag", flag), ("b_host_composed", host), ("c_device_composed", device)):
        fn()                                      # warm-up
        times[name] = [round(timed(stream, fn), 3) for _ in range(reps)]
    agree = all(all(np.array_equal(x, y) for x, y in zip(res["a"], res[arm_])) for arm_ in ("b", "c"))
    med = {k: round(statistics.median(v), 3) for k, v in times.items()}
    return {"queries": nq, "hits": hits, "documents_listed": ndocs,
            "minus_documents": int((res["a"][2] >> 31).sum()),
            "count_plus_fetch_ms_median": med, "count_plus_fetch_ms_all": times,
            "flag_over_device_composed": round(med["a_flag"] / med["c_device_composed"], 3),
            "flag_over_host_composed": round(med["a_flag"] / med["b_host_composed"], 3),
            "agree": bool(agree)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workloads", default="pangenome,documents_1kB")
    a = ap.parse_args()
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    s = stream.cuda_stream
    ctx = _lib.Context(0)
    out = {"gpu": name, "power_limit": power, "reps": a.reps}
    names = a.workloads.split(",")
    rng = np.random.default_rng(1)
    if "pangenome" in names:
        base = gen.dna(100_000)
        text, starts = copies(base, 1000, rng, 0.01, 0.001)
        arm = Arm(ctx, s, text, starts)
        guides = [g.tobytes() + b"NGG" for g in samples(base, rng, 1000, 20)]
        primers = [p.tobytes() for p in samples(base, rng, 10_000, 22)]
        res = {"n": len(text), "docs": len(starts), "genome": 100_000}
        for wname, qs, kf in (("guides_1k_x20_NGG_iupac_both_hamming_k3", guides, 3 | IUPAC | BOTH),
                              ("guides_1k_x20_NGG_iupac_both_edit_k2", guides, 2 | EDIT | IUPAC | BOTH),
                              ("primers_10k_x22_both_hamming_k2", primers, 2 | BOTH)):
            res[wname] = run(arm, stream, qs, kf, a.reps)
            print("pangenome", wname, res[wname]["count_plus_fetch_ms_median"], file=sys.stderr, flush=True)
        out["pangenome_1000_copies_100kB"] = res
        del arm
        torch.cuda.empty_cache()
    if "documents_1kB" in names:
        n = 100_000_000
        text = gen.dna(n)
        starts = cut(n, 500, 1500, 1)
        arm = Arm(ctx, s, text, starts)
        reads = [r.tobytes() for r in reads_with_indels(text, rng, 100_000, 150, 0.01, 0.005)]
        res = {"n": n, "docs": len(starts)}
        res["reads_100k_x150_edit_k4_best0"] = run(arm, stream, reads, 4 | EDIT | BEST, a.reps)
        print("documents_1kB", res["reads_100k_x150_edit_k4_best0"]["count_plus_fetch_ms_median"], file=sys.stderr,
              flush=True)
        out["documents_1kB"] = res
        del arm
        torch.cuda.empty_cache()
    rows = [r for w in out.values() if isinstance(w, dict) for r in w.values() if isinstance(r, dict)]
    out["agree"] = all(r["agree"] for r in rows)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
