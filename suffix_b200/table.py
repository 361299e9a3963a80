"""Host-side mirror of the reference's `SuffixTable` (src/table.rs:54-294).

Construction (`SuffixTable(text)` == `SuffixTable::new`, src/table.rs:78-85)
and `lcp_lens` (src/table.rs:130-138) call the CUDA library through the
C-ABI; the bookkeeping and the O(m log n) queries stay on the host exactly
like the reference (src/table.rs:197-293).
"""
import threading

import numpy as np

from . import _lib

_lock = threading.Lock()


def _as_bytes(text) -> bytes:
    if isinstance(text, str):
        return text.encode("utf-8")          # byte-level, like `Utf8` (src/table.rs:778-800)
    if isinstance(text, (bytes, bytearray, memoryview)):
        return bytes(text)
    return np.ascontiguousarray(text, dtype=np.uint8).tobytes()


class SuffixTable:
    """A sequence of lexicographically sorted suffixes (u32 byte offsets)."""

    def __init__(self, text, *, device: int = 0, _table=None):
        """SuffixTable::new (src/table.rs:78-85): O(n) construction on the GPU.
        Raises if the text exceeds B200SA_MAX_N = 2^32-4096 bytes (the reference panics above 2^32-1, :380)."""
        self._text = _as_bytes(text)
        self._device = device
        if _table is not None:
            self._table = _table
            return
        if len(self._text) > 0xFFFFF000:   # B200SA_MAX_N
            raise OverflowError("text longer than 2^32-4096 bytes (B200SA_MAX_N)")
        t = np.frombuffer(self._text, dtype=np.uint8)
        with _lock:                           # default context is not thread-safe
            ctx = _lib.default_context(device)
            self._table = ctx.build(t)
            self._stats = ctx.stats()

    # src/table.rs:111-119
    @classmethod
    def from_parts(cls, text, table) -> "SuffixTable":
        tb = _as_bytes(text)
        table = np.ascontiguousarray(table, dtype=np.uint32)
        assert len(tb) == len(table), "text and table lengths differ"   # assert_eq!, :117
        return cls(tb, _table=table)

    # src/table.rs:125-127
    def into_parts(self):
        return self._text, self._table

    # src/table.rs:130-138 (semantics of lcp_lens_quadratic, :348-361)
    def lcp_lens(self) -> np.ndarray:
        t = np.frombuffer(self._text, dtype=np.uint8)
        with _lock:
            return _lib.default_context(self._device).lcp(t, self._table)

    def table(self) -> np.ndarray:            # :142-144
        return self._table

    def text(self) -> bytes:                  # :148-150 (bytes; the reference returns &str)
        return self._text

    def __len__(self) -> int:                 # :156-158
        return len(self._table)

    def len(self) -> int:
        return len(self._table)

    def is_empty(self) -> bool:               # :162-164
        return len(self._table) == 0

    def suffix(self, i: int) -> str:          # :168-170
        return self._text[int(self._table[i]):].decode("utf-8")

    def suffix_bytes(self, i: int) -> bytes:  # :174-176
        return self._text[int(self._table[i]):]

    def __eq__(self, other):                  # derived PartialEq, :54
        return isinstance(other, SuffixTable) and self._text == other._text and \
            np.array_equal(self._table, other._table)

    # ---- queries (host side, like the reference)
    def contains(self, query) -> bool:        # :197-199
        return self.any_position(query) is not None

    def positions(self, query) -> np.ndarray:
        """src/table.rs:223-259: sub-slice of the table (SA order, unsorted)."""
        text, q = self._text, _as_bytes(query)
        n, tab = len(text), self._table
        empty = tab[0:0]
        if n == 0 or len(q) == 0:
            return empty
        m = len(q)
        # bounded heads instead of whole suffixes: `q <= text[s..]` <=> `q <= text[s..s+m]`
        # (O(m) per probe, no copy of the suffix -- like the reference's slice compares)
        h0 = text[int(tab[0]):int(tab[0]) + m]
        hl = text[int(tab[n - 1]):int(tab[n - 1]) + m]
        if q < h0 or q > hl:                  # :228-235 (q < s0 && !s0.starts_with(q)) || q > last
            return empty
        lo, hi = 0, n                         # binary_search, :900-914
        while lo < hi:
            mid = (lo + hi) // 2
            s = int(tab[mid])
            if q <= text[s:s + m]:
                hi = mid
            else:
                lo = mid + 1
        start = lo
        lo, hi = 0, n - start
        while lo < hi:
            mid = (lo + hi) // 2
            if not text.startswith(q, int(tab[start + mid])):
                hi = mid
            else:
                lo = mid + 1
        end = start + lo
        return empty if start > end else tab[start:end]

    def any_position(self, query):
        """src/table.rs:279-293: some position of `query`, or None."""
        text, q = self._text, _as_bytes(query)
        if len(q) == 0:
            return None
        tab = self._table
        lo, hi = 0, len(tab)
        m = len(q)
        while lo < hi:
            mid = (lo + hi) // 2
            s = int(tab[mid])
            head = text[s:s + m]
            if head == q:
                return s
            if head < q:
                lo = mid + 1
            else:
                hi = mid
        return None

    # ---- LCP-interval tree (SURVEY 8f-4; the node set of the reference's suffix tree,
    # suffix_tree/src/lib.rs:392-505): (psv, nsv) per rank from b200sa_lcp_intervals_dev
    def lcp_intervals(self, lcp=None):
        """Returns (lcp, psv, nsv): the internal node owning the boundary before rank i is the
        interval [psv[i], nsv[i]) of string depth lcp[i] (psv == 0xFFFFFFFF: none to the left)."""
        import torch
        lcp = self.lcp_lens() if lcp is None else np.ascontiguousarray(lcp, dtype=np.uint32)
        n = len(lcp)
        dev = torch.device("cuda", self._device)
        d_l = torch.from_numpy(lcp.astype(np.int64)).to(dev).to(torch.int32)
        d_p = torch.empty(n, dtype=torch.int32, device=dev)
        d_n = torch.empty(n, dtype=torch.int32, device=dev)
        with _lock:
            _lib.default_context(self._device).lcp_intervals_dev(d_l.data_ptr(), n, d_p.data_ptr(), d_n.data_ptr(),
                                                                 torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return lcp, d_p.cpu().numpy().view(np.uint32), d_n.cpu().numpy().view(np.uint32)

    # ---- matching statistics and SMEMs (DESIGN 6b f-10)
    def _device_arrays(self):
        """Device copies of the text, the table and lcp_lens(), made on first use and kept while the table
        lives: 9 bytes per text byte of device memory."""
        if getattr(self, "_dev", None) is None:
            import torch
            dev = torch.device("cuda", self._device)
            up = lambda a: torch.from_numpy(a.copy()).to(dev)
            lcp = self.lcp_lens()
            self._dev = (up(np.frombuffer(self._text or b"\0", dtype=np.uint8)),
                         up(np.ascontiguousarray(self._table, dtype=np.uint32).view(np.int32)),
                         up(lcp.view(np.int32)))
        return self._dev

    def _match_call(self, ctx, d_q, d_off, nq, q_bytes, d_len, d_start, d_end, stream):
        d_t, d_sa, d_lcp = self._dev
        ctx.match_stats_dev(d_t.data_ptr(), len(self._table), d_sa.data_ptr(), d_lcp.data_ptr(), d_q, d_off, nq,
                            q_bytes, d_len, d_start, d_end, stream)

    def matching_statistics(self, queries):
        """For every byte of every query, the longest piece starting there that occurs in the text, and
        where (b200sa_match_stats_dev): (offsets u64[nq + 1], length u32[], start u32[], end u32[]), the
        row of query q, offset j at offsets[q] + j.  length is the longest l with query[j:j + l] in the
        text; table()[start:end] are its occurrences, what positions(query[j:j + l]) returns ((0, 0) when
        l = 0).  Uses _device_arrays()."""
        from . import _match
        self._device_arrays()
        return _match.matching_statistics(self, queries)

    def smems(self, queries, min_len=1):
        """The super-maximal exact matches of every query: its matches of at least min_len bytes that lie
        inside no other match of the same query (b200sa_smems_dev).  (offsets u64[nq + 1], qpos u32[],
        length u32[], start u32[], end u32[]): query q's rows are [offsets[q], offsets[q+1]) by ascending
        qpos, the match is query[qpos:qpos + length] and table()[start:end] are its occurrences."""
        from . import _match
        self._device_arrays()
        return _match.smems(self, queries, min_len)

    # ---- repeats (DESIGN 6b f-11)
    _REPEAT_MODES = ("any", "earlier")

    def _repeat_arrays(self):
        _, d_sa, d_lcp = self._device_arrays()
        return d_sa, d_lcp, None, 0

    def repeat_lengths(self) -> np.ndarray:
        """u32[n]: for every position p, the longest prefix of text[p:] that also starts at another
        position (b200sa_repeat_lens_dev).  Uses _device_arrays()."""
        from . import _repeats
        return _repeats.repeat_lengths(self)

    def repeated_substrings(self, min_len, with_ends=False):
        """The distinct strings of min_len bytes that occur at least twice, as ranges of the table
        (b200sa_repeat_runs_dev): (start u32[], end u32[]) in ascending order, table()[start:end] the
        occurrences of one string, what positions() returns for it.  with_ends adds (first u32[], last
        u32[]), the smallest and largest of those positions."""
        from . import _repeats
        return _repeats.repeated_substrings(self, min_len, with_ends)

    def duplicate_spans(self, min_len, mode="any"):
        """(begin u32[], end u32[]): the maximal spans of bytes covered by a flagged position's next
        min_len bytes, by ascending begin (b200sa_duplicate_spans_dev).  mode "any" flags every position
        whose next min_len bytes occur at another position, "earlier" every such occurrence but the
        first."""
        from . import _repeats
        return _repeats.duplicate_spans(self, min_len, mode, self._REPEAT_MODES)

    def duplicated_bytes(self, min_len, mode="any") -> int:
        """The number of bytes duplicate_spans(min_len, mode) covers, without fetching the spans."""
        from . import _repeats
        return _repeats.duplicated_bytes(self, min_len, mode, self._REPEAT_MODES)

    # ---- longest previous factor and LZ77 (DESIGN 6b f-12)
    def longest_previous_factors(self):
        """(lpf u32[n], src u32[n]): lpf[p] is the longest prefix of text[p:] that also starts at some
        q < p (the occurrence may overlap p); src[p] is one such q, 0xFFFFFFFF where lpf[p] = 0
        (b200sa_lpf_dev).  src is an earlier occurrence, not necessarily the leftmost or the closest."""
        from . import _lz
        return _lz.longest_previous_factors(self)

    def lz77_factors(self, *, _cap_guess=None):
        """(start u32[z], length u32[z], source u32[z]): the LZ77 factorization of the text, the greedy
        parse by longest previous factors (b200sa_lz77_dev).  A factor of length l at start copies
        text[source:source + l] (source < start, the copy may overlap); a literal has length 1 and
        source 0xFFFFFFFF and stands for the byte text[start]."""
        from . import _lz
        return _lz.lz77_factors(self, _cap_guess)

    def lz77_count(self) -> int:
        """z, the number of LZ77 factors, without fetching them."""
        from . import _lz
        return _lz.lz77_count(self)

    # ---- Burrows-Wheeler transform (DESIGN 6b f-13)
    def _bwt_arrays(self):
        """Device copies of the text and the table: those of _device_arrays() when they exist, else made
        on first use without the LCP array and kept while the table lives (5 bytes per text byte)."""
        if getattr(self, "_dev", None) is not None:
            return self._dev[0], self._dev[1], None, 0
        if getattr(self, "_dev_bwt", None) is None:
            import torch
            dev = torch.device("cuda", self._device)
            up = lambda a: torch.from_numpy(a.copy()).to(dev)
            self._dev_bwt = (up(np.frombuffer(self._text or b"\0", dtype=np.uint8)),
                             up(np.ascontiguousarray(self._table, dtype=np.uint32).view(np.int32)))
        return self._dev_bwt[0], self._dev_bwt[1], None, 0

    def bwt(self):
        """(bwt bytes[n], primary): the Burrows-Wheeler transform of text + $, with $ below every byte and
        left out of the bytes; primary is the row of $, 1 + the rank of position 0 (b200sa_bwt_dev).
        suffix_b200.inverse_bwt(bwt, primary) gives the text back."""
        from . import _bwt
        b, term = _bwt.bwt(self)
        return b, int(term[0])

    def bwt_runs(self) -> int:
        """r, the number of maximal runs of equal symbols in the transform's n + 1 symbols, $ included."""
        from . import _bwt
        return _bwt.bwt_runs(self)

    # ---- approximate positions (DESIGN 6b f-14 .. f-18, f-20, f-21)
    def approximate_positions(self, query, k, *, metric="hamming", best=None, iupac=False, strands="forward",
                              fixed=False, bulges=None, loci=False):
        """(positions u32[], mismatches u32[]): every p with p + m <= n where text[p:p + m] differs from
        the query (m bytes) in at most k bytes, 0 <= k <= 31, by ascending p, with that number of
        mismatches beside it (b200sa_approx_positions_dev).  b"" matches nothing; for k = 0 the positions
        are those of positions(query), sorted.  Uses the device copies of _bwt_arrays().
        metric="edit": every p in [0, n) with dist(p) <= k instead, dist(p) the least Levenshtein distance
        between the query and a text[p:e], e <= n, listed beside p; an exact hit at p also puts its neighbours
        at distance 1 (include/b200sa.h, B200SA_APPROX_EDIT).  Any other metric than "hamming" or "edit" raises
        ValueError.
        best=s (an int, 0 <= s <= 31) lists only each query's best hits: with best(q) its least distance within
        k, the occurrences at distance <= min(k, best(q) + s), exactly what the call returns at that threshold
        (B200SA_APPROX_BEST).  best=0 gives each query's best hits, and the distance column then holds best(q)
        on every one.  best=None (the default) lists every occurrence within k; any other value, True included,
        raises ValueError.
        iupac=True reads each query byte as an IUPAC nucleotide code (A C G T, U = T, R Y S W K M B D H V N, in
        either case), which matches the uppercase text bytes A C G T of its class (B200SA_APPROX_IUPAC); any
        other query byte raises B200SA_ERR_BAD_ARG.  Lowercase (soft-masked) text bases, N, U and every other
        text byte match no code and count as a mismatch: uppercase a soft-masked text before building the
        table.  Combines with metric= and best=; a non-bool value raises ValueError.
        fixed=True (with iupac=True; a non-bool value, or fixed=True without iupac=True, raises ValueError) keeps
        the lowercase symbols of each query fixed (B200SA_APPROX_FIXED, the text going through
        b200sa_docs_approx_positions_dev as one document on a SuffixTable): a lowercase code still means its
        uppercase class, but must match it, and takes no substitution, insertion or adjacent deletion, so the
        threshold is spent on the uppercase symbols alone.  A CRISPR guide written "GACGCTGACGCTGACGCTGAngg"
        finds off-targets whose PAM is intact, with mismatches and bulges in the spacer only.  A query with no
        lowercase symbol gives exactly the call without the flag.
        bulges=(dna, rna) (two ints in 0 .. 3; needs metric="edit", best=None and k + dna + rna <= 31; any
        other value than None raises ValueError) searches as CRISPR off-target tools do, with three budgets in
        place of one (B200SA_APPROX_BULGES, the text going through b200sa_docs_approx_positions_dev as one
        document on a SuffixTable): p is listed when some alignment of the query to a text[p:e] has at most k
        substitutions, at most dna DNA bulges (text bases with no query base) and at most rna RNA bulges (query
        bases with no text base), with the least total of the three over those alignments beside it.
        bulges=(0, 0) gives exactly the Hamming call; combines with iupac=, fixed= and strands=.
        loci=True (a non-bool value raises ValueError) lists one hit per locus in place of the run of
        neighbouring starts that one site yields (B200SA_APPROX_LOCI (the text going through b200sa_docs_approx_positions_dev as one document on a
        SuffixTable)): a locus is a
        chain of hits on one strand whose consecutive starts are less than the query's length
        apart, and its hit with the least distance, the leftmost on a tie, represents it.  So a planted site gives
        one hit under metric="edit" and bulges= as under Hamming, and approximate_counts counts sites.  The result
        is a subset of the call without it, at equal distances; combines with every other keyword.
        strands="both" also lists the occurrences of the query's reverse complement (A <-> T, C <-> G in either
        case; with iupac=True each code's class complemented, R <-> Y, K <-> M, B <-> V, D <-> H, U -> A) as
        minus-strand hits at the leftmost text position of their window or alignment
        (B200SA_APPROX_BOTH_STRANDS), and returns (positions, distances, minus): one list by (p, strand) with
        the plus hit first, minus a bool array; with best= best(q) is taken over both strands.  strands="forward"
        (the default) searches the query alone; any other value raises ValueError."""
        from . import _approx
        return _approx.positions(self, query, k, metric, best, iupac, strands, fixed, bulges, loci)

    def approximate_positions_batch(self, queries, k, *, metric="hamming", best=None, iupac=False, strands="forward",
                                    fixed=False, bulges=None, loci=False):
        """(offsets u64[nq + 1], positions u32[], mismatches u32[]): query q's occurrences with at most k
        mismatches (or within k edits, metric="edit") are positions[offsets[q]:offsets[q + 1]], as
        approximate_positions returns them; best=0 gives each query's best hits, with best(q) in the
        distance column (best=, iupac=, fixed=, bulges= and loci= as in approximate_positions).  strands="both" returns (offsets,
        positions, distances, minus) with both strands in each query's list, as approximate_positions does."""
        from . import _approx
        return _approx.positions_batch(self, queries, k, metric, best, iupac, strands, fixed, bulges, loci)

    def approximate_counts(self, queries, k, *, metric="hamming", best=None, iupac=False, strands="forward",
                           fixed=False, bulges=None, loci=False):
        """u64[nq]: the number of occurrences with at most k mismatches (or within k edits, metric="edit") of
        every query, without fetching them; best=0 counts each query's best hits, those at distance best(q)
        (best=, iupac=, fixed= and bulges= as in approximate_positions); strands="both" counts the hits of both strands;
        loci=True counts loci, the sites that approximate_positions(loci=True) lists."""
        from . import _approx
        return _approx.counts(self, queries, k, metric, best, iupac, strands, fixed, bulges, loci)

    def approximate_alignments(self, query, k, *, metric="hamming", best=None, iupac=False, strands="forward"):
        """(positions u32[], distances u32[], ends u32[], cigar_offsets u64[h + 1], cigar u32[]): the hits of
        approximate_positions, in its order, each with its alignment (B200SA_APPROX_ALIGN on
        b200sa_docs_approx_positions_dev, the text as one document, computed on the device).  Hit i aligns the query to text[positions[i]:ends[i]]; its operations are
        cigar[cigar_offsets[i]:cigar_offsets[i + 1]], BAM words len << 4 | code (I 1, D 2, = 7, X 8), in text
        order; suffix_b200.cigar_string turns them into "12=1X7=".  With metric="edit" the alignment is the
        canonical walk of include/b200sa.h, which prefers a substitution or match, then an insertion, then a
        deletion; the query must then be at most 4096 bytes (B200SA_APPROX_ALIGN_MAX_M).  distances and ends are
        read off the operations.  strands="both" returns (positions, distances, minus, ends, cigar_offsets,
        cigar), and a minus hit's operations align the reverse complement, as SAM does.  Keywords are checked as
        in approximate_positions."""
        from . import _approx
        return _approx.alignments(self, query, k, metric, best, iupac, strands)

    def approximate_alignments_batch(self, queries, k, *, metric="hamming", best=None, iupac=False,
                                     strands="forward"):
        """(offsets u64[nq + 1], positions, distances, ends, cigar_offsets, cigar): query q's hits are
        [offsets[q], offsets[q + 1]) of positions, distances and ends, as approximate_alignments returns them;
        one count call, then one fetch call sized by it.  strands="both" puts minus after distances."""
        from . import _approx
        return _approx.alignments_batch(self, queries, k, metric, best, iupac, strands)

    # ---- persistence (SURVEY 8f-2): the only "wire format" the reference API implies is
    # from_parts/into_parts (src/table.rs:111-127): text bytes + little-endian u32 table.
    def save(self, path: str) -> None:
        """Writes `<path>.text` (raw bytes) and `<path>.sa` (raw little-endian u32)."""
        with open(path + ".text", "wb") as f:
            f.write(self._text)
        self._table.astype("<u4").tofile(path + ".sa")

    @classmethod
    def load(cls, path: str, mmap: bool = True) -> "SuffixTable":
        """from_parts over files written by save(); the table is memory-mapped by default."""
        with open(path + ".text", "rb") as f:
            text = f.read()
        table = np.memmap(path + ".sa", dtype="<u4", mode="r") if mmap else np.fromfile(path + ".sa", dtype="<u4")
        assert len(text) == len(table), "text and table lengths differ"
        return cls(text, _table=table)

    def last_stats(self) -> dict:
        return getattr(self, "_stats", {})

    def __repr__(self):
        return "SuffixTable(n=%d)" % len(self._table)
