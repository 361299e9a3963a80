"""Host statement of top-k document retrieval (include/b200sa.h, b200sa_docs_topk_dev) on top of the listing
of tests/model_docs_list.py: its entries (d, tf) sorted by (-tf, d), the first min(k, df) kept."""
from tests import model_docs_list


def top_k(starts, n, doc, byd, prev, s, e, k):
    """[(d, tf), ...] of the range [s, e): tf descending, ties by ascending document."""
    rows = [(d, tf) for _, d, tf in model_docs_list.listing(starts, n, doc, byd, prev, s, e)]
    rows.sort(key=lambda r: (-r[1], r[0]))
    return rows[:k]
