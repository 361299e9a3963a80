"""f-8: document listing (b200sa_docs_list_index_dev, b200sa_docs_list_dev) against the occurrence route on
the device.  Prints one JSON line: card and power limit; the median CUDA-event time of the index build
(one warm-up, then --reps); per batch the median times of the listing (with tf) and of the occurrence
route (gather G over the ranges, b200sa_doc_ids_dev, torch.unique of (query, document)), alternated, the
listed entries and occurrences, the phase split of one timed listing call, and whether both routes give
the same (query, document, count) rows; the device workspace of an index build plus the largest batch
on a fresh context in bytes per text byte.

    python tools/docs_list_bench.py [--n 100000000] [--reps 5]

Text: G_dna cut into documents of about 1 kB (500..1499 bytes, tools/docs_bench.cut).  Batches: (a)
100,000 random 12-mers of the text, (b) 10,000 random 8-mers, (c) the four one-byte queries, (d) (a) +
(c).  G comes from b200sa_docs_build_dev and the ranges from b200sa_docs_positions_dev, all on the device;
the ranges are found once per batch and are not part of either route's time."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _lib, gen
from tools.docs_bench import card, cut, phase_times, timed


def kmers(text, k, count, seed):
    rng = np.random.default_rng(seed)
    return [text[a:a + k].tobytes() for a in rng.integers(0, len(text) - k, count)]


def ranges(ctx, s, d_t, d_g, d_s, ndocs, qs):
    off = np.zeros(len(qs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(q) for q in qs])
    d_q = torch.from_numpy(np.frombuffer(b"".join(qs), np.uint8).copy()).cuda()
    d_off = torch.from_numpy(off.view(np.int64)).cuda()
    d_start = torch.empty(len(qs), dtype=torch.int32, device="cuda")
    d_end = torch.empty(len(qs), dtype=torch.int32, device="cuda")
    ctx.docs_positions_dev(d_t.data_ptr(), len(d_t), d_g.data_ptr(), d_s.data_ptr(), ndocs, d_q.data_ptr(),
                           d_off.data_ptr(), len(qs), d_start.data_ptr(), d_end.data_ptr(), s)
    torch.cuda.synchronize()
    return d_start, d_end


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
    starts = cut(n, 500, 1500, 1)
    ndocs = len(starts)
    d_t = torch.from_numpy(text).cuda()
    d_s = torch.from_numpy(starts.view(np.int32).copy()).cuda()
    d_g = torch.empty(n, dtype=torch.int32, device="cuda")
    ctx.docs_build_dev(d_t.data_ptr(), n, d_s.data_ptr(), ndocs, d_g.data_ptr(), 0, s)
    byd = torch.empty(n, dtype=torch.int32, device="cuda")
    prev = torch.empty(n, dtype=torch.int32, device="cuda")

    def index(c=ctx):
        c.docs_list_index_dev(n, d_g.data_ptr(), d_s.data_ptr(), ndocs, byd.data_ptr(), prev.data_ptr(), s)

    index()
    t_index = [timed(stream, index) for _ in range(a.reps)]
    ctx.set_timing(True)
    index()
    index_phases = {p: round(ms, 3) for p, ms in phase_times(ctx)}
    ctx.set_timing(False)
    out = {"gpu": name, "power_limit": power, "text": "G_dna", "n": n, "docs": ndocs,
           "index_dev_ms_median": round(statistics.median(t_index), 3), "index_dev_ms_all": [round(x, 3) for x in t_index],
           "index_phases_ms": index_phases}

    a12 = kmers(text, 12, 100_000, 2)
    batches = {"kmer12_100k": a12, "kmer8_10k": kmers(text, 8, 10_000, 3), "one_byte_4": [b"A", b"C", b"G", b"T"],
               "kmer12_100k_plus_one_byte": a12 + [b"A", b"C", b"G", b"T"]}
    for bname, qs in batches.items():
        nq = len(qs)
        d_start, d_end = ranges(ctx, s, d_t, d_g, d_s, ndocs, qs)
        d_off = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
        buf = {}

        def listing(cap):
            return ctx.docs_list_dev(n, d_g.data_ptr(), d_s.data_ptr(), ndocs, byd.data_ptr(), prev.data_ptr(),
                                     d_start.data_ptr(), d_end.data_ptr(), nq, d_off.data_ptr(),
                                     buf["docs"].data_ptr() if cap else 0, buf["tf"].data_ptr() if cap else 0, cap, s)

        buf["docs"] = buf["tf"] = None
        total = listing(0)
        buf["docs"] = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")
        buf["tf"] = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")
        lens = (d_end.long() - d_start.long())
        occ = int(lens.sum())
        res = {}

        def occurrences():
            qid = torch.repeat_interleave(torch.arange(nq, device="cuda"), lens, output_size=occ)
            first = torch.cumsum(lens, 0) - lens
            rank = torch.arange(occ, device="cuda") - first[qid] + d_start.long()[qid]
            pos = d_g[rank]
            doc = torch.empty(occ, dtype=torch.int32, device="cuda")
            off = torch.empty(occ, dtype=torch.int32, device="cuda")
            ctx.doc_ids_dev(pos.data_ptr(), occ, d_s.data_ptr(), ndocs, doc.data_ptr(), off.data_ptr(), s)
            res["keys"], res["counts"] = torch.unique((qid << 32) | doc.long(), return_counts=True)

        listing(total)
        occurrences()
        tl, to = [], []
        for _ in range(a.reps):                  # alternated, so both see the same card state
            tl.append(timed(stream, lambda: listing(total)))
            to.append(timed(stream, occurrences))
        ctx.set_timing(True)
        listing(total)
        phases = {p: round(ms, 3) for p, ms in phase_times(ctx)}
        ctx.set_timing(False)
        # agreement: the listing sorted by (query, document) equals the unique (query, document) rows
        q = torch.repeat_interleave(torch.arange(nq, device="cuda"), d_off.diff())
        key = (q << 32) | (buf["docs"][:total].long() & 0xFFFFFFFF)
        order = torch.argsort(key)
        agree = (total == len(res["keys"]) and bool(torch.equal(key[order], res["keys"])) and
                 bool(torch.equal(buf["tf"][:total][order].long(), res["counts"])))
        out[bname] = {"queries": nq, "listed": total, "occurrences": occ,
                      "list_dev_ms_median": round(statistics.median(tl), 3), "list_dev_ms_all": [round(x, 3) for x in tl],
                      "occurrence_route_ms_median": round(statistics.median(to), 3),
                      "occurrence_route_ms_all": [round(x, 3) for x in to], "list_phases_ms": phases, "agree": agree}
        del res, buf

    fresh = _lib.Context(0)                      # workspace of an index build and the largest batch
    index(fresh)
    qs = batches["kmer12_100k_plus_one_byte"]
    d_start, d_end = ranges(fresh, s, d_t, d_g, d_s, ndocs, qs)
    d_off = torch.empty(len(qs) + 1, dtype=torch.int64, device="cuda")
    fresh.docs_list_dev(n, d_g.data_ptr(), d_s.data_ptr(), ndocs, byd.data_ptr(), prev.data_ptr(), d_start.data_ptr(),
                        d_end.data_ptr(), len(qs), d_off.data_ptr(), 0, 0, 0, s)
    torch.cuda.synchronize()
    out["workspace_bytes_per_text_byte"] = round(fresh.stats()["workspace_bytes"] / n, 1)
    fresh.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
