"""Matching statistics and SMEMs over a device-resident table: the part SuffixTable and
DocumentSuffixTable share.  A table supplies `_device` and `_match_call(ctx, d_q, d_off, nq, q_bytes,
d_len, d_start, d_end, stream)`, its own b200sa_*match_stats_dev call."""
import numpy as np

from . import _lib
from .table import _as_bytes, _lock


def _stats_dev(table, queries):
    """(offsets u64 on the host, d_off, d_len, d_start, d_end): the arrays left on the device as int32
    tensors of u32 values (int64 for the offsets)."""
    import torch
    qs = [_as_bytes(q) for q in queries]
    nq = len(qs)
    dev = torch.device("cuda", table._device)
    off = np.zeros(nq + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(q) for q in qs])
    q_bytes = int(off[nq])
    d_off = torch.from_numpy(off.view(np.int64)).to(dev)
    d_len, d_start, d_end = (torch.empty(q_bytes, dtype=torch.int32, device=dev) for _ in range(3))
    if q_bytes:
        d_q = torch.from_numpy(np.frombuffer(b"".join(qs), dtype=np.uint8).copy()).to(dev)
        with _lock:
            table._match_call(_lib.default_context(table._device), d_q.data_ptr(), d_off.data_ptr(), nq, q_bytes,
                              d_len.data_ptr(), d_start.data_ptr(), d_end.data_ptr(),
                              torch.cuda.current_stream(dev).cuda_stream)
        torch.cuda.synchronize(dev)
    return off, d_off, d_len, d_start, d_end


def _host(t):
    return t.cpu().numpy().view(np.uint32)


def matching_statistics(table, queries):
    off, _, d_len, d_start, d_end = _stats_dev(table, queries)
    return off, _host(d_len), _host(d_start), _host(d_end)


def smems(table, queries, min_len):
    import torch
    min_len = int(min_len)
    if min_len < 1:
        raise ValueError("min_len must be at least 1, got %d" % min_len)
    off, d_off, d_len, d_start, d_end = _stats_dev(table, queries)
    nq, q_bytes = len(off) - 1, int(off[-1])
    dev = d_off.device
    d_so = torch.zeros(nq + 1, dtype=torch.int64, device=dev)
    ctx = _lib.default_context(table._device)
    stream = torch.cuda.current_stream(dev).cuda_stream
    with _lock:                                   # count, then fetch into a buffer of that size
        total = ctx.smems_dev(d_off.data_ptr(), nq, q_bytes, d_len.data_ptr(), min_len, d_so.data_ptr(), 0, 0, stream)
        qpos = torch.empty(total, dtype=torch.int32, device=dev)
        if total:
            ctx.smems_dev(d_off.data_ptr(), nq, q_bytes, d_len.data_ptr(), min_len, d_so.data_ptr(), qpos.data_ptr(),
                          total, stream)
    at = torch.repeat_interleave(d_off[:-1], d_so.diff()) + qpos      # the pattern position of every SMEM
    torch.cuda.synchronize(dev)
    return d_so.cpu().numpy().view(np.uint64), _host(qpos), _host(d_len[at]), _host(d_start[at]), _host(d_end[at])
