"""f-9: top-k document retrieval (b200sa_docs_topk_dev) against the listing route on the device.  Prints one
JSON line: card and power limit; per workload the median CUDA-event times (one warm-up, then --reps,
alternated) of top-k and of the listing route (b200sa_docs_list_dev with tf, one device sort of the entries
by (query, -tf, document), a per-query cut to k), the listed entries, the phase split of one timed top-k
call (phases of all rounds summed), and whether both routes give the same rows; the device workspace of
top-k on the largest batch, on a fresh context.

    python tools/docs_topk_bench.py [--n 100000000] [--reps 5]

Text: G_dna cut into documents of about 1 kB (500..1499 bytes), as tools/docs_list_bench.py, and n/4
copies of ACGT.  The workloads put queries on both sides of each size-class threshold of docs_topk.cuh
(df <= 32: one warp; <= 4096: one block; larger: levels of tiles): random 12-mers (df about 7) and 10-mers
(about 95); 8-mers (about 1.5 k) and 7-mers (about 6 k); all 4,096 6-mers (about 22 k) at k = 10 and 1,024;
the four one-byte queries (about 100 k); b"A" on the ACGT copies (n/4); and the 6-mers again with a round
budget of 2^22 entries (B200SA_TOPK_ROUND), to show what rounds cost.  Ranges come from
b200sa_docs_positions_dev once per workload and are in neither route's time."""
import argparse
import itertools
import json
import os
import statistics
import sys

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _lib, gen
from tools.docs_bench import card, cut, phase_times, timed
from tools.docs_list_bench import kmers, ranges


class Table:
    """G, byd and prev of one document set, device-resident."""

    def __init__(self, ctx, s, text, starts):
        self.n, self.ndocs = len(text), len(starts)
        self.d_t = torch.from_numpy(text).cuda()
        self.d_s = torch.from_numpy(starts.view(np.int32).copy()).cuda()
        self.d_g = torch.empty(self.n, dtype=torch.int32, device="cuda")
        ctx.docs_build_dev(self.d_t.data_ptr(), self.n, self.d_s.data_ptr(), self.ndocs, self.d_g.data_ptr(), 0, s)
        self.byd = torch.empty(self.n, dtype=torch.int32, device="cuda")
        self.prev = torch.empty(self.n, dtype=torch.int32, device="cuda")
        ctx.docs_list_index_dev(self.n, self.d_g.data_ptr(), self.d_s.data_ptr(), self.ndocs, self.byd.data_ptr(),
                                self.prev.data_ptr(), s)
        torch.cuda.synchronize()

    def args(self):
        return (self.n, self.d_g.data_ptr(), self.d_s.data_ptr(), self.ndocs, self.byd.data_ptr(), self.prev.data_ptr())


def run(ctx, s, stream, tab, qs, k, reps, env=None):
    nq = len(qs)
    d_start, d_end = ranges(ctx, s, tab.d_t, tab.d_g, tab.d_s, tab.ndocs, qs)
    count = torch.empty(nq, dtype=torch.int32, device="cuda")
    tdocs = torch.empty(nq * k, dtype=torch.int32, device="cuda")
    ttf = torch.empty(nq * k, dtype=torch.int32, device="cuda")

    def topk():
        ctx.docs_topk_dev(*tab.args(), d_start.data_ptr(), d_end.data_ptr(), nq, k, count.data_ptr(),
                          tdocs.data_ptr(), ttf.data_ptr(), s)

    d_off = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
    total = ctx.docs_list_dev(*tab.args(), d_start.data_ptr(), d_end.data_ptr(), nq, d_off.data_ptr(), 0, 0, 0, s)
    ldocs = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")
    ltf = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")
    res = {}
    db = max(1, int(tab.ndocs - 1).bit_length())
    qb = max(1, nq.bit_length())

    def route():
        ctx.docs_list_dev(*tab.args(), d_start.data_ptr(), d_end.data_ptr(), nq, d_off.data_ptr(), ldocs.data_ptr(),
                          ltf.data_ptr(), total, s)
        tf = ltf[:total].long()
        tmax = int(tf.max()) if total else 0
        tb = max(1, tmax.bit_length())
        assert qb + tb + db <= 63
        q = torch.repeat_interleave(torch.arange(nq, device="cuda"), d_off.diff(), output_size=total)
        key = (q << (tb + db)) | ((tmax - tf) << db) | ldocs[:total].long()
        key, order = torch.sort(key)
        j = torch.arange(total, device="cuda") - d_off[:-1][q]   # q is ascending, so rank within the query
        keep = j < k
        res["docs"], res["tf"] = (key[keep] & ((1 << db) - 1)).int(), ltf[:total][order][keep]

    old = {v: os.environ.get(v) for v in (env or {})}
    os.environ.update(env or {})
    try:
        topk()
        route()
        tt, tr = [], []
        for _ in range(reps):                    # alternated, so both see the same card state
            tt.append(timed(stream, topk))
            tr.append(timed(stream, route))
        ctx.set_timing(True)
        topk()
        phases = {}
        for p, ms in phase_times(ctx):
            phases[p] = round(phases.get(p, 0.0) + ms, 3)
        rounds = [p for p, _ in phase_times(ctx)].count("topk_emit")
        ctx.set_timing(False)
    finally:
        for v, x in old.items():
            if x is None:
                del os.environ[v]
            else:
                os.environ[v] = x
    torch.cuda.synchronize()
    keep = torch.arange(k, device="cuda", dtype=torch.int32)[None, :] < count[:, None]
    agree = (bool(torch.equal(count.long(), torch.clamp(d_off.diff(), max=k))) and
             bool(torch.equal(tdocs.view(nq, k)[keep], res["docs"])) and
             bool(torch.equal(ttf.view(nq, k)[keep], res["tf"])))
    return {"queries": nq, "k": k, "listed": total, "rows": int(count.sum()), "rounds": rounds,
            "topk_ms_median": round(statistics.median(tt), 3), "topk_ms_all": [round(x, 3) for x in tt],
            "listing_route_ms_median": round(statistics.median(tr), 3), "listing_route_ms_all": [round(x, 3) for x in tr],
            "topk_phases_ms": phases, "agree": agree}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    s = stream.cuda_stream
    ctx = _lib.Context(0)
    n = a.n
    text = gen.dna(n)
    dna = Table(ctx, s, text, cut(n, 500, 1500, 1))
    out = {"gpu": name, "power_limit": power, "text": "G_dna", "n": n, "docs": dna.ndocs}
    six = [bytes(x) for x in itertools.product(b"ACGT", repeat=6)]
    work = [("kmer12_100k_k10", kmers(text, 12, 100_000, 2), 10, None),
            ("kmer10_20k_k10", kmers(text, 10, 20_000, 4), 10, None),
            ("kmer8_10k_k10", kmers(text, 8, 10_000, 3), 10, None),
            ("kmer7_2k_k10", kmers(text, 7, 2_000, 5), 10, None),
            ("kmer6_all_k10", six, 10, None),
            ("kmer6_all_k1024", six, 1024, None),
            ("one_byte_4_k10", [b"A", b"C", b"G", b"T"], 10, None),
            ("kmer6_all_k10_round_4M", six, 10, {"B200SA_TOPK_ROUND": str(1 << 22)})]
    for wname, qs, k, env in work:
        out[wname] = run(ctx, s, stream, dna, qs, k, a.reps, env)

    fresh = _lib.Context(0)                      # workspace of top-k on the largest batch
    d_start, d_end = ranges(fresh, s, dna.d_t, dna.d_g, dna.d_s, dna.ndocs, six)
    buf = torch.empty(len(six) * 1024 * 2 + len(six), dtype=torch.int32, device="cuda")
    p = buf.data_ptr()
    fresh.docs_topk_dev(*dna.args(), d_start.data_ptr(), d_end.data_ptr(), len(six), 1024, p, p + 4 * len(six),
                        p + 4 * len(six) * 1025, s)
    torch.cuda.synchronize()
    out["workspace_bytes_kmer6_all_k1024"] = fresh.stats()["workspace_bytes"]
    fresh.close()
    del dna
    torch.cuda.empty_cache()

    acgt = np.frombuffer(b"ACGT" * (n // 4), dtype=np.uint8).copy()
    copies = Table(ctx, s, acgt, np.arange(0, len(acgt), 4, dtype=np.uint32))
    out["acgt_copies_A_k10"] = run(ctx, s, stream, copies, [b"A"], 10, a.reps)
    out["acgt_copies_A_k10"]["docs"] = copies.ndocs
    print(json.dumps(out))


if __name__ == "__main__":
    main()
