"""Exact k-mer counts for any k up to 31 (EXTENSION).

The reference counts k-mers exactly only for k <= 8, where the table has 4^k bins (kmer_encodings.py:72-74).  Here the
distinct k-mers and their counts live in an open-addressing hash table in device memory, filled by the row-driven
k-mer kernel (``bnpk_rows_kmer_table_insert``): what ``jellyfish count`` produces
(benchmarks/rules/kmer_counting.smk:1-31).

    counts = bnp.count_kmers_exact(chunk.sequence, 31)               # -> KmerCounts
    counter = bnp.KmerCounter(31, canonical=True)                     # streaming
    for chunk in bnp.open("reads.fq.gz").read_chunks():
        counter.add(chunk.sequence)
    counts = counter.result()
    counts.kmers, counts.counts                                       # int64 CUDA tensors, kmers ascending

A k-mer is its hash ``sum_j code[i+j] * 4^j`` (as ``get_kmers``); with ``canonical=True`` the smaller of that and the
hash of its reverse complement (as ``get_kmers(..., canonical=True)``).

Memory: 16 bytes per slot (int64 key + int64 count), and the table is kept at most half full (``MAX_LOAD``), so 32 bytes
or more per distinct k-mer.  Growing it rehashes into a table of twice (or more) the slots while the old one still
exists; ``result()`` needs another 16 bytes per distinct k-mer for the sorted copy."""
import torch

from .. import _native as nv
from .. import ops
from ..encoded_array import EncodedArray, EncodedRaggedArray
from ..encodings.exceptions import EncodingError
from ..streams import _is_stream
from ..rows import LONG_ROW
from .kmers import _source_of, rescan_kmers

MAX_LOAD = 0.5            # keys per slot the table may reach; every insert launch stays within it
MIN_BATCH = 1 << 20       # k-mer positions: grow rather than launch on less free room than this
DEFAULT_CAPACITY = 1 << 16  # expected distinct k-mers when the caller gives no capacity


def table_limit(slots: int) -> int:
    """Keys a table of ``slots`` slots may hold."""
    return int(slots * MAX_LOAD)


def slots_for(n_keys: int) -> int:
    """The smallest power-of-two table that holds ``n_keys`` keys within the load limit."""
    slots = 2
    while table_limit(slots) < n_keys:
        slots *= 2
    return slots


def plan_insert(offsets, row: int, done: int, total: int, n_used: int, slots: int, min_batch: int = MIN_BATCH):
    """The next launch of adding rows ``[row, R)`` to a table of ``slots`` slots that holds ``n_used`` keys.

    ``offsets`` (int64[R+1], on any device) are the exclusive prefix sums of the rows' k-mer positions, ``done`` =
    offsets[row] and ``total`` = offsets[R].  Every position may be a new key, so a launch of rows ``[row, end)`` may
    claim up to ``offsets[end] - done`` slots.  Returns ``(slots', end, offsets[end])``: grow the table to ``slots'``
    slots first (``slots' == slots``: no growth), then insert rows ``[row, end)``; then
    ``n_used + offsets[end] - done <= MAX_LOAD * slots'`` and ``end > row`` (for ``row < R``).

    All remaining rows go in one launch when they fit.  Otherwise the table grows (doubling) until the free room holds
    ``min(remaining positions, min_batch)`` and the first row, and the launch takes the longest run of rows that fits."""
    n_rows = offsets.numel() - 1
    if n_used + (total - done) <= table_limit(slots):
        return slots, n_rows, total
    while table_limit(slots) - n_used < min(total - done, min_batch):
        slots *= 2
    target = torch.tensor([done + table_limit(slots) - n_used], dtype=offsets.dtype, device=offsets.device)
    end = torch.searchsorted(offsets, target, right=True) - 1
    end, end_pos, first_end = torch.cat([end, offsets[end], offsets[row + 1:row + 2]]).tolist()
    if end <= row:                      # the first row alone is larger than the free room
        while table_limit(slots) - n_used < first_end - done:
            slots *= 2
        end, end_pos = row + 1, first_end
    return slots, end, end_pos


class KmerCounts:
    """Distinct k-mers and how often each occurred: ``kmers`` ascending, ``counts`` > 0 (int64 CUDA tensors)."""

    def __init__(self, kmers, counts, k: int, alphabet_encoding, canonical: bool = False):
        self.kmers, self.counts = kmers, counts
        self.k, self.alphabet_encoding, self.canonical = k, alphabet_encoding, canonical

    def __len__(self):
        return self.kmers.numel()

    def __repr__(self):
        return f"KmerCounts(k={self.k}, distinct={len(self)}, canonical={self.canonical})"

    def _hash_of(self, kmer: str) -> int:
        letters = self.alphabet_encoding.get_alphabet()
        if len(kmer) != self.k:
            raise ValueError(f"{kmer!r} is not a {self.k}-mer")
        try:
            codes = [letters.index(c.upper()) for c in kmer]
        except ValueError:
            raise ValueError(f"{kmer!r} has letters outside {''.join(letters)}") from None
        h = sum(c << (2 * j) for j, c in enumerate(codes))
        if self.canonical:
            from .dna import complement_xor_of
            x = complement_xor_of(self.alphabet_encoding)
            h = min(h, sum((c ^ x) << (2 * j) for j, c in enumerate(reversed(codes))))
        return h

    def get_counts(self, kmers):
        """Counts of k-mers given as strings (turned into canonical hashes for a canonical table) or as hash values
        (looked up as they are); 0 for k-mers that did not occur.  Returns an int64 tensor."""
        if isinstance(kmers, str):
            kmers = [kmers]
        if isinstance(kmers, (list, tuple)) and kmers and isinstance(kmers[0], str):
            kmers = [self._hash_of(s) for s in kmers]
        q = torch.as_tensor(kmers, dtype=torch.int64).to(self.kmers.device).reshape(-1)
        if len(self) == 0:
            return torch.zeros_like(q)
        idx = torch.searchsorted(self.kmers, q).clamp_(max=len(self) - 1)
        return torch.where(self.kmers[idx] == q, self.counts[idx], torch.zeros_like(q))

    def __getitem__(self, kmer: str) -> int:
        return int(self.get_counts([kmer])[0].item())

    def most_common(self, n: int = None):
        """(kmers, counts) by count descending, equal counts by k-mer ascending."""
        order = torch.sort(self.counts, descending=True, stable=True).indices
        if n is not None:
            order = order[:n]
        return self.kmers[order], self.counts[order]

    def spectrum(self, max_count: int):
        """int64[max_count + 1]: bin c = distinct k-mers seen c times; the last bin counts those seen max_count times or
        more (bin 0 is 0)."""
        if max_count < 1:
            raise ValueError("max_count must be positive")
        clipped = torch.clamp(self.counts, max=max_count).contiguous()
        return ops.bincount(clipped, max_count + 1)[0]


class KmerCounter:
    """Streaming exact k-mer counter: ``add`` sequences (any number of chunks), then ``result()``.

    ``capacity`` is the number of distinct k-mers expected; it sizes the first table (default: grow from
    DEFAULT_CAPACITY).  A bad base raises ``EncodingError`` with the offset ``get_kmers`` reports on the same input; as
    that launch's k-mers are already in the table, the counter then refuses further ``add`` and ``result`` calls."""

    def __init__(self, k: int, canonical: bool = False, capacity: int = None):
        assert 0 < k < 32, "k must be larger than 0 and smaller than 32"
        self.k, self.canonical = k, canonical
        self._slots = slots_for(DEFAULT_CAPACITY if capacity is None else max(int(capacity), 1))
        self._keys = self._counts = self._state = None
        self._alphabet = None
        self._cxor = 0
        self._n_used = 0
        self._error = None
        self.n_grows = 0

    @property
    def capacity(self) -> int:
        """Slots of the table (of the first table before the first ``add``)."""
        return self._slots

    @property
    def table_bytes(self) -> int:
        return 16 * self._slots

    @property
    def n_distinct(self) -> int:
        return self._n_used

    def _raise_if_failed(self):
        if self._error is not None:
            raise RuntimeError(f"this KmerCounter failed earlier and holds partial counts: {self._error}") from self._error

    def _new_table(self, slots, device):
        return (torch.full((slots,), -1, dtype=torch.int64, device=device),
                torch.zeros(slots, dtype=torch.int64, device=device))

    def _status(self):
        """The status block (first ST_WORDS words of the state; the last word is n_used), re-initialised."""
        return ops.reset_status(self._state[:nv.ST_WORDS])

    def _read_state(self):
        words = self._state.tolist()
        self._n_used = words[nv.ST_WORDS]
        if words[nv.ST_TABLE_FULL]:
            self._error = RuntimeError("k-mer table overflowed (the load limit was not kept): counts are incomplete")
            raise self._error
        return words

    def _grow(self, slots):
        dev = self._keys.device
        keys, counts = self._new_table(slots, dev)
        before = self._n_used
        self._state[nv.ST_WORDS] = 0
        ops.kmer_table_rehash(self._keys, self._counts, keys, counts, self._state[nv.ST_WORDS:], status=self._status())
        self._keys, self._counts, self._slots = keys, counts, slots
        self._read_state()
        if self._n_used != before:
            self._error = RuntimeError(f"k-mer table rehash kept {self._n_used} of {before} keys")
            raise self._error
        self.n_grows += 1

    def add(self, sequence):
        """Count the k-mers of ``sequence``: an EncodedRaggedArray / 1-D EncodedArray of BaseEncoding text (read as
        DNAEncoding) or of a four-letter AlphabetEncoding, or a record chunk with a ``sequence`` field."""
        self._raise_if_failed()
        if hasattr(sequence, "sequence") and not isinstance(sequence, (EncodedArray, EncodedRaggedArray)):
            sequence = sequence.sequence
        src = _source_of(sequence)
        enc = src.alphabet_encoding
        if enc.alphabet_size != 4:
            raise NotImplementedError("exact k-mer counts are only implemented for four-letter alphabets")
        if self._alphabet is None:
            if self.canonical:
                from .dna import complement_xor_of
                self._cxor = complement_xor_of(enc)
            self._alphabet = enc
            self._keys, self._counts = self._new_table(self._slots, src.base.device)
            self._state = torch.zeros(nv.ST_WORDS + 1, dtype=torch.int64, device=src.base.device)
        elif enc != self._alphabet:
            raise ValueError(f"KmerCounter counts {self._alphabet} k-mers, got {enc}")
        elif src.base.device != self._keys.device:
            raise ValueError(f"KmerCounter lives on {self._keys.device}, got a sequence on {src.base.device}")
        if src.lens.numel():
            self._insert(src)
        return self

    def _insert(self, rows):
        k = self.k
        offsets = ops.row_offsets(rows.lens, k - 1)
        total, longest = torch.stack([offsets[-1], rows.lens.max().to(torch.int64)]).tolist()
        pieces = rows
        if longest > LONG_ROW + k - 1:
            # chromosome-length rows: pieces of LONG_ROW positions, one warp each (same positions, same total)
            pieces = rows.split(k)[0]
            offsets = ops.row_offsets(pieces.lens, k - 1)
        n_used_t = self._state[nv.ST_WORDS:]
        row, done = 0, 0
        while row < pieces.lens.numel():
            slots, end, end_pos = plan_insert(offsets, row, done, total, self._n_used, self._slots, MIN_BATCH)
            if slots != self._slots:
                self._grow(slots)
            ops.rows_kmer_table_insert(rows.base, pieces.starts[row:end], pieces.lens[row:end], rows.enc_mode, k,
                                       self._keys, self._counts, n_used_t, self._cxor, rows.lut, status=self._status())
            words = self._read_state()
            if words[nv.ST_BAD_BASE] != nv.INT64_MAX:
                try:
                    rows.raise_bad_base(self._state[:nv.ST_WORDS], rescan_kmers)
                except EncodingError as e:
                    self._error = e
                    raise
            row, done = end, end_pos

    def result(self) -> KmerCounts:
        """The counts so far (the table stays usable for further ``add`` calls)."""
        self._raise_if_failed()
        alphabet = self._alphabet
        if alphabet is None:
            from ..encodings.alphabet_encoding import DNAEncoding
            empty = torch.zeros(0, dtype=torch.int64, device="cuda")
            return KmerCounts(empty, empty.clone(), self.k, DNAEncoding, self.canonical)
        keep = self._keys >= 0
        kmers, counts = self._keys[keep], self._counts[keep]
        kmers, order = torch.sort(kmers)
        return KmerCounts(kmers, counts[order], self.k, alphabet, self.canonical)


def count_kmers_exact(sequence, k: int, canonical: bool = False, capacity: int = None) -> KmerCounts:
    """EXTENSION: exact counts of the distinct k-mers of ``sequence`` (k in 1..31), see ``KmerCounter``.  A stream of
    sequences (or record chunks) is counted into one table."""
    counter = KmerCounter(k, canonical=canonical, capacity=capacity)
    if _is_stream(sequence):
        for s in sequence:
            counter.add(s)
    else:
        counter.add(sequence)
    return counter.result()
