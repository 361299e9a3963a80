"""Repeat lengths, runs and duplicate spans over a device-resident table: the part SuffixTable and
DocumentSuffixTable share.  A table supplies `_device` and `_repeat_arrays()` -> (d_table, d_lcp,
d_doc_starts or None, ndocs), its arrays on the device."""
import numpy as np

from . import _lib
from .table import _lock

MODES = {"any": 0, "earlier": 1, "other_document": 2, "earlier_document": 3}
_U32_MAX = 0xFFFFFFFF


def _host(t):
    return t.cpu().numpy().view(np.uint32)


def _min_len(min_len):
    min_len = int(min_len)
    if min_len < 1:
        raise ValueError("min_len must be at least 1, got %d" % min_len)
    return min(min_len, _U32_MAX)          # no text is that long: nothing repeats at either length


def _mode(mode, allowed):
    if mode not in allowed:
        raise ValueError("mode must be one of %s, got %r" % (", ".join(repr(m) for m in allowed), mode))
    return MODES[mode]


def _setup(table):
    import torch
    d_r, d_lcp, d_starts, ndocs = table._repeat_arrays()
    dev = torch.device("cuda", table._device)
    return (torch, dev, _lib.default_context(table._device), torch.cuda.current_stream(dev).cuda_stream, len(table),
            d_r, d_lcp, d_starts, ndocs)


def repeat_lengths(table):
    torch, dev, ctx, stream, n, d_r, d_lcp, _, _ = _setup(table)
    d_rl = torch.empty(n, dtype=torch.int32, device=dev)
    if n:
        with _lock:
            ctx.repeat_lens_dev(n, d_r.data_ptr(), d_lcp.data_ptr(), d_rl.data_ptr(), stream)
        torch.cuda.synchronize(dev)
    return _host(d_rl)


def repeated_substrings(table, min_len, with_ends):
    min_len = _min_len(min_len)
    torch, dev, ctx, stream, n, d_r, d_lcp, _, _ = _setup(table)
    with _lock:                                   # count, then fetch into buffers of that size
        total = ctx.repeat_runs_dev(n, d_r.data_ptr(), d_lcp.data_ptr(), min_len, stream=stream) if n else 0
        out = [torch.empty(total, dtype=torch.int32, device=dev) for _ in range(4 if with_ends else 2)]
        if total:
            ctx.repeat_runs_dev(n, d_r.data_ptr(), d_lcp.data_ptr(), min_len, *(o.data_ptr() for o in out), cap=total,
                                stream=stream)
    return tuple(_host(o) for o in out)


def duplicate_spans_dev(table, min_len, mode, allowed):
    """(begin, end) as device tensors, in coordinates of the text or concatenation."""
    min_len, mode = _min_len(min_len), _mode(mode, allowed)
    torch, dev, ctx, stream, n, d_r, d_lcp, d_starts, ndocs = _setup(table)
    args = (n, d_r.data_ptr(), d_lcp.data_ptr(), d_starts.data_ptr() if d_starts is not None else 0, ndocs, min_len,
            mode)
    with _lock:
        total = ctx.duplicate_spans_dev(*args, stream=stream)[0] if n else 0
        begin, end = (torch.empty(total, dtype=torch.int32, device=dev) for _ in range(2))
        if total:
            ctx.duplicate_spans_dev(*args, begin.data_ptr(), end.data_ptr(), total, stream=stream)
    return begin, end


def duplicate_spans(table, min_len, mode, allowed):
    return tuple(_host(t) for t in duplicate_spans_dev(table, min_len, mode, allowed))


def duplicated_bytes(table, min_len, mode, allowed):
    min_len, mode = _min_len(min_len), _mode(mode, allowed)
    _, _, ctx, stream, n, d_r, d_lcp, d_starts, ndocs = _setup(table)
    if not n:
        return 0
    with _lock:
        return ctx.duplicate_spans_dev(n, d_r.data_ptr(), d_lcp.data_ptr(),
                                       d_starts.data_ptr() if d_starts is not None else 0, ndocs, min_len, mode,
                                       stream=stream)[1]
