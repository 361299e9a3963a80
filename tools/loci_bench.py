"""f-23: one hit per locus (B200SA_APPROX_LOCI on b200sa_docs_approx_positions_dev, a single text as one document)
on device-resident tables.  Prints one JSON line: card and power limit, read in the same run; per arm the hits of
the call without the flag and the loci with it, the median CUDA-event time (one warm-up each, then --reps rounds
that alternate the arms) of the count call plus the fetch call with and without bit 7 and of the composed baseline,
the phase times of the flag's fetch call, and whether the flag's listing equals tests/model_loci.collapse of the
plain fetch over the whole arm, and the composed baseline's.

    python tools/loci_bench.py [--reps 5] [--arms f22,guides,reads]

The composed baseline is what a caller has without the flag, kept on the device with torch, as approx_docs_bench.py
does for f-19: the plain count and fetch, then each hit's document by searchsorted over the document starts, a sort
by (query, strand, p), the locus heads from neighbouring starts, a segment minimum of (d << 32) | p by
scatter_reduce, and the kept hits compacted with their offsets.

Arms: the f-22 off-target search (10 MB G_dna, 100 random 20-nt guides + "ngg" with the PAM fixed, both strands,
bulges (4, 1, 1)); 1 k random 20-nt guides + "NGG" under B200SA_APPROX_IUPAC at edit k = 2 on both strands over
100 MB G_dna; and 100 k reads of 150 bytes (1 % substitutions, 0.5 % insertions or deletions) at edit k = 4 with
best=0 over 100 MB G_dna, where a read's best stratum still holds the shifted starts of its one site."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _lib, gen
from tests import model_loci
from tools.approx_bench import Arm
from tools.docs_bench import card, phase_times, timed
from tools.edit_bench import reads_with_indels

LOCI, EDIT, BEST, BULGES, IUPAC, FIXED, BOTH = 0x80, 0x10000, 0x100000, 0x200000, 0x1000000, 0x2000000, 0x10000000
MINUS = 0x80000000


class Batch:
    """Queries on the device with their offsets, an offsets output and fetch buffers of the plain call's size."""

    def __init__(self, qs):
        self.nq = len(qs)
        off = np.zeros(self.nq + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(q) for q in qs])
        self.d_q = torch.from_numpy(np.frombuffer(b"".join(qs), dtype=np.uint8).copy()).cuda()
        self.d_off = torch.from_numpy(off.view(np.int64)).cuda()
        self.d_o = torch.empty(self.nq + 1, dtype=torch.int64, device="cuda")
        self.d_len = torch.from_numpy(np.diff(off.astype(np.int64))).cuda()

    def call(self, arm, kf, pos=None, dist=None, cap=0):
        return arm.approx(self.d_q.data_ptr(), self.d_off.data_ptr(), self.nq, kf, self.d_o.data_ptr(),
                          0 if pos is None else pos.data_ptr(), 0 if dist is None else dist.data_ptr(), cap)

    def fetch(self, arm, kf, pos, dist):
        """The protocol a caller follows: count, then fetch."""
        total = self.call(arm, kf)
        self.call(arm, kf, pos, dist, total)
        return total


def composed(d_o, pos, dist, d_len, d_starts, nq):
    """The collapse of the plain device listing with torch: (offsets, pos, dist) on the device."""
    q = torch.repeat_interleave(torch.arange(nq, device="cuda"), d_o.diff())
    p = pos.long() & 0xFFFFFFFF
    dl = dist.long() & 0xFFFFFFFF
    minus, d = dl >> 31, dl & (MINUS - 1)
    doc = torch.searchsorted(d_starts, p, right=True) - 1
    order = torch.argsort((q << 33) | (minus << 32) | p)
    qs, ss, ps, ds = q[order], minus[order], p[order], doc[order]
    head = torch.ones_like(qs, dtype=torch.bool)
    head[1:] = (qs[1:] != qs[:-1]) | (ss[1:] != ss[:-1]) | (ds[1:] != ds[:-1]) | (ps[1:] - ps[:-1] >= d_len[qs[1:]])
    locus = torch.cumsum(head.long(), 0) - 1
    key = (d[order] << 32) | ps
    least = torch.full((int(locus[-1]) + 1,), 1 << 62, dtype=torch.int64, device="cuda")
    least = least.scatter_reduce(0, locus, key, "amin")
    keep = torch.zeros_like(head)
    keep[order] = least[locus] == key
    o = torch.zeros(nq + 1, dtype=torch.int64, device="cuda")
    o[1:] = torch.cumsum(torch.bincount(q[keep], minlength=nq), 0)
    return o, pos[keep], dist[keep]


def host(t):
    return t.cpu().numpy()


def run(arm, stream, qs, kf, reps):
    b = Batch(qs)
    nq = len(qs)
    hits = b.call(arm, kf)
    pos = torch.empty(max(hits, 1), dtype=torch.int32, device="cuda")
    dist = torch.empty(max(hits, 1), dtype=torch.int32, device="cuda")
    lpos = torch.empty(max(hits, 1), dtype=torch.int32, device="cuda")
    ldist = torch.empty(max(hits, 1), dtype=torch.int32, device="cuda")
    d_starts = torch.from_numpy(arm.starts.astype(np.int64)).cuda()
    res = {}

    def plain():
        res["plain"] = b.fetch(arm, kf, pos, dist)
        res["plain_off"] = b.d_o.clone()

    def flag():
        res["loci"] = b.fetch(arm, kf | LOCI, lpos, ldist)
        res["loci_off"] = b.d_o.clone()

    def comp():
        b.fetch(arm, kf, pos, dist)
        res["composed"] = composed(b.d_o, pos[:hits], dist[:hits], b.d_len, d_starts, nq)

    arms = (("plain", plain), ("loci", flag), ("composed", comp))
    times = {name: [] for name, _ in arms}
    for _, fn in arms:
        fn()                                      # warm-up
    for _ in range(reps):
        for name, fn in arms:
            times[name].append(round(timed(stream, fn), 3))
    loci = res["loci"]
    got = (host(res["loci_off"]).view(np.uint64), host(lpos[:loci]).view(np.uint32), host(ldist[:loci]).view(np.uint32))
    plain_list = (host(res["plain_off"]).view(np.uint64), host(pos[:hits]).view(np.uint32),
                  host(dist[:hits]).view(np.uint32))
    want = model_loci.collapse(plain_list, qs, arm.starts)
    co = res["composed"]
    comp_list = (host(co[0]).astype(np.uint64), host(co[1]).view(np.uint32), host(co[2]).view(np.uint32))
    arm.ctx.set_timing(True)                      # a separate run: phase times of the flag's fetch call
    b.call(arm, kf | LOCI, lpos, ldist, loci)
    phases = {}
    for p, v in phase_times(arm.ctx):
        phases[p] = round(phases.get(p, 0.0) + v, 3)
    arm.ctx.set_timing(False)
    med = {k: round(statistics.median(v), 3) for k, v in times.items()}
    return {"queries": nq, "hits": hits, "loci": loci, "count_plus_fetch_ms_median": med,
            "count_plus_fetch_ms_all": times, "loci_over_plain": round(med["loci"] / med["plain"], 3),
            "loci_over_composed": round(med["loci"] / med["composed"], 3),
            "fetch_phases_ms": {p: v for p, v in phases.items() if p.startswith("loci") or p.startswith("approx")},
            "agree_model": all(np.array_equal(x, y) for x, y in zip(got, want)),
            "agree_composed": all(np.array_equal(x, y) for x, y in zip(got, comp_list))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--arms", default="f22,guides,reads")
    a = ap.parse_args()
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    ctx = _lib.Context(0)
    out = {"gpu": name, "power_limit": power, "text": "G_dna", "reps": a.reps}
    names = a.arms.split(",")
    one = np.zeros(1, dtype=np.uint32)
    if "f22" in names:
        rng = np.random.default_rng(1)
        arm = Arm(ctx, stream.cuda_stream, gen.dna(10_000_000), one)
        qs = [bytes(rng.choice(list(b"ACGT"), 20).tolist()) + b"ngg" for _ in range(100)]
        kf = 4 | (1 << 17) | (1 << 22) | BULGES | EDIT | IUPAC | FIXED | BOTH
        out["f22_10MB_guides_100_ngg_both_bulges_4_1_1"] = run(arm, stream, qs, kf, a.reps)
        print("f22", out["f22_10MB_guides_100_ngg_both_bulges_4_1_1"]["count_plus_fetch_ms_median"], file=sys.stderr,
              flush=True)
        del arm
        torch.cuda.empty_cache()
    if "guides" in names or "reads" in names:
        text = gen.dna(100_000_000)
        arm = Arm(ctx, stream.cuda_stream, text, one)
        if "guides" in names:
            rng = np.random.default_rng(2)
            qs = [bytes(rng.choice(list(b"ACGT"), 20).tolist()) + b"NGG" for _ in range(1000)]
            out["guides_1k_NGG_both_edit_k2_100MB"] = run(arm, stream, qs, 2 | EDIT | IUPAC | BOTH, a.reps)
            print("guides", out["guides_1k_NGG_both_edit_k2_100MB"]["count_plus_fetch_ms_median"], file=sys.stderr,
                  flush=True)
        if "reads" in names:
            rng = np.random.default_rng(3)
            reads = [r.tobytes() for r in reads_with_indels(text, rng, 100_000, 150, 0.01, 0.005)]
            out["reads_100k_x150_edit_k4_best0_100MB"] = run(arm, stream, reads, 4 | EDIT | BEST, a.reps)
            print("reads", out["reads_100k_x150_edit_k4_best0_100MB"]["count_plus_fetch_ms_median"], file=sys.stderr,
                  flush=True)
        del arm
        torch.cuda.empty_cache()
    rows = [r for r in out.values() if isinstance(r, dict)]
    out["agree"] = all(r["agree_model"] and r["agree_composed"] for r in rows)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
