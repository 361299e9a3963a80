"""f-20: the alignments of approximate hits (B200SA_APPROX_ALIGN on b200sa_docs_approx_positions_dev) on
device-resident tables.  Prints one JSON line: card and power limit; per table and workload the median CUDA-event
time (one warm-up, then --reps) of the count call plus the fetch call with the flag and without it, the phase split
of one fetch call with the flag, the numbers of hits and operations, and a sample of hits aligned by the serial C
statement tests/align_check.c on one host core, with its time and whether it equals the device's words.

    python tools/align_bench.py [--reps 5] [--sample 2000] [--tables text,documents_1kB]

Tables: 100 MB G_dna as one text (through the documents entry as one document, as SuffixTable does) and the same
text cut into ~1 kB documents.  Workloads: 1 k 20-nt guides + NGG under B200SA_APPROX_IUPAC on both strands at
Hamming k = 3 and edit k = 2 (off-target scoring needs the mismatch positions), and 100 k reads of 150 bytes with
1 % substitutions and 0.5 % insertions or deletions at edit k = 4, with and without best=0 (read mapping needs a
CIGAR)."""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _approx, _lib, gen
from tests import align_check
from tools.approx_bench import Arm
from tools.approx_docs_bench import Batch, samples
from tools.docs_bench import card, cut, phase_times, timed
from tools.edit_bench import reads_with_indels

EDIT, BEST, IUPAC, BOTH, ALIGN = 0x10000, 0x100000, 0x1000000, 0x10000000, 0x8000000
MINUS = 0x80000000


class DocsArm(Arm):
    """An Arm whose calls all go through the documents entry; a single text is one document."""

    def __init__(self, ctx, s, text, starts):
        super().__init__(ctx, s, text, starts)
        if starts is None:
            self.d_s = torch.zeros(1, dtype=torch.int32, device="cuda")
            self.starts = np.zeros(1, dtype=np.uint32)

    def approx(self, d_q, d_off, nq, k, d_o, d_pos=0, d_mis=0, cap=0):
        return self.ctx.docs_approx_positions_dev(self.d_t.data_ptr(), self.n, self.d_sa.data_ptr(),
                                                  self.d_s.data_ptr(), len(self.starts), d_q, d_off, nq, k, d_o,
                                                  d_pos, d_mis, cap, self.s)


def run(arm, ctx, stream, qs, kf, reps, sample, rng):
    one = Batch(qs)
    ka = kf | ALIGN
    ops = one.call(arm, ka)
    hits = one.call(arm, kf)
    wpos = torch.empty(max(ops, 1), dtype=torch.int32, device="cuda")
    words = torch.empty(max(ops, 1), dtype=torch.int32, device="cuda")
    pos = torch.empty(max(hits, 1), dtype=torch.int32, device="cuda")
    dist = torch.empty(max(hits, 1), dtype=torch.int32, device="cuda")
    res = {}

    def flag():                                   # the protocol a caller follows: count, then fetch
        one.call(arm, ka)
        one.call(arm, ka, wpos, words, ops)
        res["align"] = (one.d_o.cpu().numpy().view(np.uint64).copy(), wpos[:ops].cpu().numpy().view(np.uint32),
                        words[:ops].cpu().numpy().view(np.uint32))

    def plain():                                  # the hits alone
        one.call(arm, kf)
        one.call(arm, kf, pos, dist, hits)
        res["plain"] = (one.d_o.cpu().numpy().view(np.uint64).copy(), pos[:hits].cpu().numpy().view(np.uint32),
                        dist[:hits].cpu().numpy().view(np.uint32))

    times = {}
    for name, fn in (("align", flag), ("plain", plain)):
        fn()                                      # warm-up
        times[name] = [round(timed(stream, fn), 3) for _ in range(reps)]
    ctx.set_timing(True)
    one.call(arm, ka, wpos, words, ops)
    phases = {}
    for nm, ms in phase_times(ctx):
        phases[nm] = round(phases.get(nm, 0.0) + ms, 3)
    ctx.set_timing(False)
    # the hits read back from the listing must be the plain call's
    hoff, hp, hd, minus, _, coff, cig = _approx._hits(*res["align"])
    hd = hd | np.where(minus, np.uint32(MINUS), np.uint32(0))
    same_hits = all(np.array_equal(x, y) for x, y in zip((hoff, hp, hd), res["plain"]))
    # a sample aligned on one host core
    pick = np.sort(rng.choice(len(hp), min(sample, len(hp)), replace=False)) if len(hp) else np.zeros(0, np.int64)
    hq = np.repeat(np.arange(len(qs)), np.diff(hoff.astype(np.int64)))[pick]
    t0 = time.perf_counter()
    _, w = align_check.align_hits(arm.text, arm.starts, qs, hq, hp[pick], hd[pick], kf & EDIT, kf & IUPAC)
    host_s = time.perf_counter() - t0
    dev_w = np.concatenate([cig[int(coff[i]):int(coff[i + 1])] for i in pick]) if len(pick) else cig[:0]
    med = {k: round(statistics.median(v), 3) for k, v in times.items()}
    return {"queries": len(qs), "hits": hits, "operations": ops,
            "count_plus_fetch_ms_median": med, "count_plus_fetch_ms_all": times,
            "align_over_plain": round(med["align"] / med["plain"], 3), "align_fetch_phase_ms": phases,
            "host_sample_hits": int(len(pick)), "host_sample_s": round(host_s, 3),
            "host_sample_us_per_hit": round(1e6 * host_s / max(len(pick), 1), 2),
            "agree": bool(same_hits and np.array_equal(dev_w, w & np.uint32(MINUS - 1)))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=2000)
    ap.add_argument("--tables", default="text,documents_1kB")
    a = ap.parse_args()
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    s = stream.cuda_stream
    ctx = _lib.Context(0)
    out = {"gpu": name, "power_limit": power, "reps": a.reps}
    n = 100_000_000
    text = gen.dna(n)
    rng = np.random.default_rng(1)
    guides = [g.tobytes() + b"NGG" for g in samples(text, rng, 1000, 20)]
    reads = [r.tobytes() for r in reads_with_indels(text, rng, 100_000, 150, 0.01, 0.005)]
    for table in a.tables.split(","):
        arm = DocsArm(ctx, s, text, None if table == "text" else cut(n, 500, 1500, 1))
        res = {"n": n, "docs": len(arm.starts)}
        for wname, qs, kf in (("guides_1k_x20_NGG_iupac_both_hamming_k3", guides, 3 | IUPAC | BOTH),
                              ("guides_1k_x20_NGG_iupac_both_edit_k2", guides, 2 | EDIT | IUPAC | BOTH),
                              ("reads_100k_x150_edit_k4", reads, 4 | EDIT),
                              ("reads_100k_x150_edit_k4_best0", reads, 4 | EDIT | BEST)):
            res[wname] = run(arm, ctx, stream, qs, kf, a.reps, a.sample, rng)
            print(table, wname, res[wname]["count_plus_fetch_ms_median"], file=sys.stderr, flush=True)
        out[table] = res
        del arm
        torch.cuda.empty_cache()
    rows = [r for w in out.values() if isinstance(w, dict) for r in w.values() if isinstance(r, dict)]
    out["agree"] = all(r["agree"] for r in rows)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
