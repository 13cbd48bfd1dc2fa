"""get_transcript_sequences (mirror of bionumpy/sequence/genes.py): the spliced sequence of every transcript of GTF/GFF
entries, built on the device with three synchronisations whatever the number of transcripts.

  exons      : gtf_entries.get_exons() (one synchronisation: the exon count and the first missing attribute).
  grouping   : a transcript is a run of consecutive exons with equal transcript_id (bnpk_rows_equal_prev), in file
               order, as the reference's itertools.groupby; its strand is its first exon's.
  order      : each transcript's exons sorted by start, ascending for '+' and '.', descending for '-'
               (lexsort_order), so that gathering every exon of a '-' transcript reverse-complemented gives the
               reverse complement of the exons joined in ascending order.  The reference joins exons in file order,
               which reverses GENCODE's '-' transcripts (their exons are listed 5' to 3', descending).
  gather     : one bnpk_interval_gather of every exon (one synchronisation: the output size), from an indexed FASTA by
               each exon's chromosome or from one 1-D sequence, with a complement table for both cases.
  bases      : one bnpk_rows_encode pass through a table that upper-cases ACGTN and rejects every other byte (one
               synchronisation); a bad byte raises EncodingError with its flat offset in the output, as the reference's
               ACGTnEncoding does."""
import numpy as np
import torch

from .. import _native as nv
from .. import config
from .. import ops
from ..arithmetics.intervals import lexsort_order, to_device
from ..datatypes import SequenceEntry
from ..encoded_array import BaseEncoding, EncodedArray, EncodedRaggedArray, as_encoded_array
from ..encodings import EncodingError
from ..rows import RowView

_tables = {}


def _device_tables(device):
    """(complement uint8[256], upper-case ACGTN uint8[256] with 255 for any other byte), built once per device.  The
    complement maps both cases and leaves every other byte as it is, so the base check still finds it."""
    if device not in _tables:
        comp = np.arange(256, dtype=np.uint8)
        upper = np.full(256, 255, dtype=np.uint8)
        for a, b in zip("ACGTN", "TGCAN"):
            comp[ord(a)], comp[ord(a.lower())] = ord(b), ord(b.lower())
            upper[ord(a)] = upper[ord(a.lower())] = ord(a)
        _tables[device] = (to_device(comp, device), to_device(upper, device))
    return _tables[device]


def _empty(device):
    text = EncodedRaggedArray(EncodedArray(torch.zeros(0, dtype=torch.uint8, device=device), BaseEncoding),
                              torch.zeros(0, dtype=torch.int32, device=device))
    return SequenceEntry(text, text)


def get_transcript_sequences(gtf_entries, reference_sequence) -> SequenceEntry:
    """SequenceEntry(transcript_id, sequence) of every transcript of ``gtf_entries`` (GTFEntry / GFFEntry records):
    its exons joined in ascending start order, reverse-complemented as a whole on the '-' strand, in upper-case ACGTN
    (lower-case input is accepted).  ``reference_sequence`` is an IndexedFasta (bnp.open_indexed), where each exon is
    looked up by its chromosome, or one 1-D sequence (text or an EncodedArray of text) that every exon indexes.  Starts
    are used as written, as in the reference.  An unknown chromosome raises KeyError, an exon outside its sequence
    ValueError and a byte other than ACGTN (either case) inside an exon EncodingError."""
    from ..io.indexed_fasta import IndexedFasta
    if len(gtf_entries) == 0:
        return _empty(config.default_device())
    exons = gtf_entries.get_exons()
    if len(exons) == 0:
        return _empty(exons.start.device)
    start, stop = exons.start.to(torch.int64).contiguous(), exons.stop.to(torch.int64).contiguous()
    dev = start.device
    tid = RowView(exons.transcript_id)
    new = 1 - ops.rows_equal_prev(tid.base, tid.starts, tid.lens).to(torch.int64)
    group = torch.cumsum(new, 0) - 1
    row = torch.arange(new.numel(), device=dev)
    first = torch.cummax(row * new, 0).values                      # each exon's transcript's first exon
    minus = exons.strand.raw().to(torch.int64)[first] == 1
    order = lexsort_order(torch.where(minus, -start, start), group)
    start, stop, group = start[order].contiguous(), stop[order].contiguous(), group[order]
    strand = minus[order].to(torch.uint8).contiguous()
    comp, upper = _device_tables(dev)
    extra = [new.sum()]
    if isinstance(reference_sequence, IndexedFasta):
        _, text, name_offsets, contigs = reference_sequence._name_table()
        names = RowView(exons.chromosome)
        ids, st_names = ops.name_lookup(names.base, names.starts, names.lens, text, name_offsets)
        ids, file, extra = ids[order].contiguous(), reference_sequence._file, extra + [st_names]
    else:
        seq = as_encoded_array(reference_sequence) if isinstance(reference_sequence, str) else reference_sequence
        if not isinstance(seq, EncodedArray) or not seq.encoding.is_base_encoding() or seq.raw().dim() != 1:
            raise TypeError("reference_sequence must be an IndexedFasta or one 1-D text sequence")
        ids, contigs, file = None, None, seq.raw().to(torch.uint8).contiguous()
    out, row_lens, bad, words = ops.interval_gather(file, start, stop, ids, contigs, strand, comp, extra=extra)
    n_tx = words[0]
    if len(words) > 1 and words[1].fault is not None:
        raise KeyError(exons.chromosome[words[1].fault].to_string())
    if bad is not None:
        r = int(order[bad])
        raise ValueError(f"exon {r} ({exons.chromosome[r].to_string()}:{int(exons.start[r])}-{int(exons.stop[r])}) "
                         "is not inside the reference sequence")
    tx_first = torch.nonzero_static(new, size=n_tx).reshape(-1)
    tx_lens = torch.zeros(n_tx, dtype=torch.int64, device=dev).index_add_(0, group, row_lens.to(torch.int64))
    tx_starts = (torch.cumsum(tx_lens, 0) - tx_lens).contiguous()
    tx_lens = tx_lens.to(torch.int32)
    bases, _, status = ops.rows_encode(out, tx_starts, tx_lens, nv.ENC_LUT, upper, total=out.numel())
    offset = ops.read_status(status).bad_base_offset(tx_lens)
    if offset is not None:
        raise EncodingError(f"Error when encoding to ACGTnEncoding. Invalid character at flat offset {offset}", offset)
    sequences = EncodedRaggedArray(EncodedArray(bases, BaseEncoding), tx_lens)
    return SequenceEntry(exons.transcript_id[tx_first], sequences)
