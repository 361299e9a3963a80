"""Count phases of the 2-bit induce passes on the bench text (B200SA_STEPLOG=1).

For every big step of k_induce6 (and every cascade step, listed apart) the step timeline of
block 0 gives: the count sweep (step start -> IND_MARK 1), the first grid sync (IND_MARK 1 -> 2)
and the rest of the step (offsets, scatter, second grid sync, next peek).  Big steps are split by
their source: chain lists of both passes and the L-part lists of the S pass read `sa` and its
carried words; the LMS lists of the L pass gather the text.  The sum of count + first sync over the
`sa`-sourced big steps caps what a consumer that gets its per-tile counts from the producers could
save.  Times are medians per step over R builds (the step sequence of one text is fixed), with
the min-max of the per-build sum.  Then the per-block view (as tools/blocklog.py) of the largest
`sa`-sourced big step of each pass.

usage: python tools/count_phase.py [n] [R]
"""
import os
import subprocess
import sys

os.environ["B200SA_STEPLOG"] = "1"
sys.path.insert(0, os.getcwd())
import numpy as np  # noqa: E402
import torch  # noqa: E402
from suffix_b200 import _lib, gen  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000_000
R = int(sys.argv[2]) if len(sys.argv) > 2 else 5
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
except OSError:
    pass
t = gen.dna(n)

# per-byte L counts and LMS counts (T[n-1] is L; equal neighbours share the type of the right one)
tt = torch.from_numpy(t).cuda().to(torch.int16)
cmp = torch.sign(tt[1:] - tt[:-1])                         # +1: S, -1: L, 0: same as i+1
idx = torch.where(cmp != 0, torch.arange(n - 1, device="cuda"), torch.full_like(cmp, n - 1, dtype=torch.int64))
nxt = torch.flip(torch.cummin(torch.flip(idx, [0]), 0).values, [0])
cmpx = torch.cat([cmp, torch.tensor([-1], device="cuda", dtype=cmp.dtype)])
is_s = torch.cat([cmpx[nxt] > 0, torch.tensor([False], device="cuda")])
lms = torch.zeros(n, dtype=torch.bool, device="cuda")
lms[1:] = is_s[1:] & ~is_s[:-1]
lcnt = torch.bincount(tt.long()[~is_s], minlength=256).cpu().numpy()
lmscnt = torch.bincount(tt.long()[lms], minlength=256).cpu().numpy()
del tt, cmp, idx, nxt, cmpx, is_s, lms
lms_lens = set(int(x) for x in lmscnt if x > 0)
lpart_lens = set(int(lcnt[c]) for c in range(1, 256) if lcnt[c] > 0)

ctx = _lib.Context(0)
d_t = torch.from_numpy(t).cuda()
d_sa = torch.empty(n, dtype=torch.int32, device="cuda")
blocks = torch.cuda.get_device_properties(0).multi_processor_count * 3
cascade = blocks * 2048


def build():
    ctx.build_dev(d_t.data_ptr(), n, d_sa.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def timeline():
    """[(pass, bigcount, kind, len, count_us, sync1_us, rest_us)] of the last build."""
    raw = ctx.debug_fetch(7, 8192).view(np.uint64)
    k = int(raw[0])
    rec = raw[1:1 + 2 * k].reshape(-1, 2).astype(np.int64)
    rows = []
    pas, big, i = 0, 0, 0
    while i < k - 1:
        code = int(rec[i, 1])
        if code >> 28 == 0xF:
            i += 1
            continue
        if code == 0 and pas == 0:       # the L pass logs one record without a list when it ends
            pas, big = 1, 0
            i += 1
            continue
        j = i + 1
        marks = {}
        while j < k and int(rec[j, 1]) >> 28 == 0xF:
            marks[int(rec[j, 1]) & 0xff] = int(rec[j, 0])
            j += 1
        if j >= k:
            break
        if 1 in marks and 2 in marks:      # big or cascade step (small episodes log no marks)
            ln = code
            if pas == 0 and ln in lms_lens:
                kind = "lms"
            elif pas == 1 and ln in lpart_lens:
                kind = "lpart"
            elif ln > cascade:
                kind = "chain"
            else:
                kind = "cascade"
            t0 = int(rec[i, 0])
            rows.append((pas, big, kind, ln, (marks[1] - t0) / 1e3, (marks[2] - marks[1]) / 1e3,
                         (int(rec[j, 0]) - marks[2]) / 1e3))
            big += 1
        i = j
    return rows


build()                                  # warm-up
runs = []
for _ in range(R):
    build()
    runs.append(timeline())
if any([r[:4] for r in x] != [r[:4] for r in runs[0]] for x in runs):
    sys.exit("the step sequence differs between builds")
t_med = np.median(np.array([[r[4:] for r in x] for x in runs]), axis=0)     # [step][count, sync1, rest]
rows = [r[:4] + tuple(t_med[s]) for s, r in enumerate(runs[0])]

print("n=%d blocks=%d cascade<=%d builds=%d (medians per step)" % (n, blocks, cascade, R))
print("pass big  kind        len   tiles  count_us sync1_us  rest_us")
for r in rows:
    print("%4s %3d %7s %10d %6d %9.1f %8.1f %8.1f" % ("LS"[r[0]], r[1], r[2], r[3], (r[3] + 2047) // 2048, r[4], r[5], r[6]))
tot = {}
for r in rows:
    a = tot.setdefault((r[0], r[2]), [0, 0.0, 0.0, 0.0])
    a[0] += 1; a[1] += r[4]; a[2] += r[5]; a[3] += r[6]
print("pass    kind steps count_us sync1_us  rest_us")
for key in sorted(tot):
    a = tot[key]
    print("%4s %7s %5d %8.1f %8.1f %8.1f" % ("LS"[key[0]], key[1], a[0], a[1], a[2], a[3]))
sa_src = [s for s, r in enumerate(rows) if r[2] in ("chain", "lpart")]
per_build = [sum(x[s][4] + x[s][5] for s in sa_src) for x in runs]
print("count + first sync over sa-sourced big steps: %.1f us per build (median of steps; builds %.1f..%.1f)"
      % (sum(rows[s][4] + rows[s][5] for s in sa_src), min(per_build), max(per_build)))

# per-block view of the largest sa-sourced big step of each pass
for p in (0, 1):
    cand = [r for r in rows if r[0] == p and r[2] in ("chain", "lpart")]
    if not cand:
        continue
    r = max(cand, key=lambda x: x[3])
    os.environ["B200SA_BLOCKLOG"] = "%d:%d" % (p, r[1])
    build()
    raw = ctx.debug_fetch(7, 16384).view(np.uint64)
    b = raw[4096:4096 + 6 * blocks].reshape(-1, 6).astype(np.int64)
    b = b[b[:, 0] > 0]
    d = (b[:, :5] - b[:, 0].min()) / 1e3
    cnt = d[:, 1] - d[:, 0]
    sc = d[:, 3] - d[:, 2]
    print("pass %s big step %d (%s, len %d): count us min %.1f med %.1f max %.1f | sync1 passed %.1f..%.1f | "
          "scatter us med %.1f max %.1f | sync2 passed %.1f..%.1f"
          % ("LS"[p], r[1], r[2], r[3], cnt.min(), np.median(cnt), cnt.max(), d[:, 2].min(), d[:, 2].max(),
             np.median(sc), sc.max(), d[:, 4].min(), d[:, 4].max()))
