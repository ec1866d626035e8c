"""
Flat-buffer FASTQ pipeline: bytes in -> trimmed / split FASTQ or FASTA bytes out, without per-read Python objects
(SURVEY.md 8(f) rows 2-3, host side).

The reference loads every read into a Python `NanoporeRead` (misc.py:151-168, nanopore_read.py:23-55), decides trims
read by read (nanopore_read.py:166-243) and formats output strings read by read (nanopore_read.py:76-147).  For
10^6-10^7 reads that host work would hide the GPU gain (SURVEY 7.3 item 3), so this module keeps reads as flat numpy
buffers end to end:

  parse_fasta(data)          FASTA bytes (multi-line records) -> FastqBatch with '+' qualities
  parse_fastq(data)          4-line FASTQ bytes -> FastqBatch (flat names / bases / qualities + offsets; bases
                             upper-cased, RNA reads detected and stored as T, exactly as NanoporeRead.__init__ does)
  end_windows(...)           the `seq[:end_size]` / `seq[-end_size:]` windows of every read as one ragged batch
  end_trim_amounts(...)      the reference's start/end trim rule applied to whole record arrays at once
  trim_end_adapters(...)     windows -> two batched engine calls -> trim amounts (a whole Phase B for fixed adapters)
  trimmed_ranges(...)        the `seq[start_trim : len - end_trim]` slice of every read (Python slice semantics)
  find_middle_hits(...)      Phase C on the trimmed reads: one cross-product submit, then only the reads with a hit
                             are masked and re-submitted (the reference's sequential masking, nanopore_read.py:210-243)
                             -- or, with PB200_DEVICE_MIDDLE=1, one adapterMiddleScan call that runs every round on
                             the device
  middle_trim_ranges(...)    hits -> the ranges the reference adds to `middle_trim_positions`
  emit(...)                  get_fastq / get_fasta of every read (split parts, numbering, --discard_middle,
                             --min_split_read_size, RNA T->U) as one bytes object, assembled with vectorised scatters
  search_adapter_sets(...)   Phase A: best start / end identity of every adapter set over the check reads' windows --
                             or, with PB200_DEVICE_SEARCH=1, one adapterSetSearch call that reduces them on the device
  trim_fastq(...)            all of the above for a fixed list of adapter sets: what `porechop -i x.fastq -o y.fastq`
                             writes once Phase A has chosen the sets
  call_barcodes(...)         determine_barcode (nanopore_read.py:399-470) on score matrices: best / second-best
                             with the reference's tie order, threshold, difference, --require_two_barcodes
  demux_fastq(...)           `porechop -i x.fastq -b dir`: trim + barcode call + one output per bin

The alignment engine is case-insensitive and maps U to T itself (Dna5 table); normalising at parse time only matters
because the reference writes the normalised bases back out.
"""
import os
import time

import numpy as np

from . import cpp_function_wrappers as W
from . import hostio
from .align import scores_from_records

_WS = np.zeros(256, dtype=bool)
_WS[[9, 10, 11, 12, 13, 28, 29, 30, 31, 32]] = True            # what str.strip() removes from an ASCII line


class FastqBatch:
    """Flat view of a FASTQ chunk: read i has name name_buf[name_off[i]:name_off[i+1]], bases
    seq[seq_off[i]:seq_off[i+1]] (upper case, RNA stored as T with rna[i] set), qualities likewise."""

    def __init__(self, name_buf, name_off, seq, seq_off, qual, qual_off, rna):
        self.name_buf, self.name_off = name_buf, name_off
        self.seq, self.seq_off, self.qual, self.qual_off, self.rna = seq, seq_off, qual, qual_off, rna
        self._names = None

    def __len__(self):
        return len(self.seq_off) - 1

    def lengths(self):
        return np.diff(self.seq_off)

    @property
    def names(self):
        if self._names is None:
            b, o = self.name_buf.tobytes(), self.name_off
            self._names = [b[o[i]:o[i + 1]].decode('ascii', 'replace') for i in range(len(self))]
        return self._names


def _strip(buf, starts, ends):
    """str.strip() of every line [starts, ends) -- vectorised; loops once per stripped character (normally 0 or 1)."""
    starts, ends = starts.copy(), ends.copy()
    while True:
        m = (ends > starts) & _WS[buf[np.maximum(ends - 1, 0)]]
        if not m.any():
            break
        ends -= m
    while True:
        m = (ends > starts) & _WS[buf[np.minimum(starts, len(buf) - 1)]]
        if not m.any():
            break
        starts += m
    return starts, ends


def parse_fastq(data):
    """data: bytes / uint8 array of 4-line FASTQ records ('@name', bases, '+', qualities).  Returns a FastqBatch.
    Lines are stripped like the reference's loader strips them (misc.py:160-166: `line.strip()`, name = header minus
    its first character); multi-line records are not supported there either.  Qualities shorter than the bases are
    padded with '+' (nanopore_read.py:34-36)."""
    buf = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
    if hostio.LIB is not None:
        return _parse_fastq_native(buf)
    if buf.size and buf[-1] != 10:
        buf = np.concatenate([buf, np.array([10], dtype=np.uint8)])
    nl = np.flatnonzero(buf == 10)
    if len(nl) % 4 != 0:
        raise ValueError('FASTQ chunk is not a whole number of 4-line records')
    n = len(nl) // 4
    z = np.zeros(0, dtype=np.uint8)
    if n == 0:
        o = np.zeros(1, dtype=np.int64)
        return FastqBatch(z, o, z, o.copy(), z, o.copy(), np.zeros(0, dtype=bool))
    starts = np.concatenate([[0], nl[:-1] + 1])            # start of every line
    starts, ends = _strip(buf, starts, nl)
    if not ((ends[0::4] > starts[0::4]) & (buf[starts[0::4]] == ord('@'))).all():
        raise ValueError('FASTQ record does not start with @')
    name_buf, name_off = _gather_ranges(buf, starts[0::4] + 1, ends[0::4])
    seq, seq_off = _gather_ranges(buf, starts[1::4], ends[1::4])
    qual, qual_off = _gather_ranges(buf, starts[3::4], ends[3::4])
    seq, rna = _normalise(seq, seq_off)
    short = np.diff(seq_off) - np.diff(qual_off)
    if (short > 0).any():
        qual, qual_off = _pad_segments(qual, qual_off, np.maximum(short, 0), ord('+'))
    return FastqBatch(name_buf, name_off, seq, seq_off, qual, qual_off, rna)


def _line_spans(buf):
    """stripped (start, length) of every line; lines end at '\\n' (the last one may be unterminated)."""
    if hostio.LIB is not None:
        return hostio.line_spans(buf)
    if buf.size == 0:
        z = np.zeros(0, dtype=np.int64)
        return z, z.copy()
    nl = np.flatnonzero(buf == 10)
    if buf[-1] != 10:
        nl = np.concatenate([nl, [len(buf)]])
    starts = np.concatenate([[0], nl[:-1] + 1])
    a, b = _strip(buf, starts, nl.copy())
    return a.astype(np.int64), (b - a).astype(np.int64)


def parse_fasta(data):
    """FASTA bytes -> FastqBatch, following the reference's loader (misc.py:123-148: lines stripped, blank lines
    skipped, a '>' line starts a record, sequence lines are concatenated; the read name is the whole header minus '>',
    porechop.py:234) and NanoporeRead.__init__ (qualities of a FASTA read are '+' * len, nanopore_read.py:33-36).
    Sequence before the first header or an empty header name is rejected here (the reference silently mangles both)."""
    buf = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
    a, ln = _line_spans(buf)
    keep = ln > 0
    a, ln = a[keep], ln[keep]
    z, o = np.zeros(0, dtype=np.uint8), np.zeros(1, dtype=np.int64)
    if len(a) == 0:
        return FastqBatch(z, o, z, o.copy(), z, o.copy(), np.zeros(0, dtype=bool))
    header = buf[a] == ord('>')
    if not header[0]:
        raise ValueError('FASTA does not start with a > line')
    if (ln[header] < 2).any():
        raise ValueError('FASTA record with an empty name')
    rec = np.cumsum(header) - 1                                  # record of every kept line
    n = int(rec[-1]) + 1
    name_buf, name_off = _gather_ranges(buf, a[header] + 1, a[header] + ln[header])
    body = ~header
    seq, _ = _gather_ranges(buf, a[body], a[body] + ln[body])    # sequence lines are already in record order
    seq_len = np.bincount(rec[body], weights=ln[body], minlength=n).astype(np.int64)
    seq_off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(seq_len, out=seq_off[1:])
    seq, rna = _normalise(seq, seq_off)
    return FastqBatch(name_buf, name_off, seq, seq_off, np.full(len(seq), ord('+'), dtype=np.uint8), seq_off.copy(), rna)


def _normalise(seq, seq_off):
    """seq.upper(); RNA if count('U') > count('T') -> stored as T (nanopore_read.py:26-31).  Returns (seq, rna)."""
    if hostio.LIB is not None:
        seq = np.ascontiguousarray(seq)
        return seq, hostio.normalise(seq, seq_off)
    lower = (seq >= ord('a')) & (seq <= ord('z'))
    seq = np.where(lower, seq - 32, seq).astype(np.uint8)
    rna = _segment_sums(seq == ord('U'), seq_off) > _segment_sums(seq == ord('T'), seq_off)
    if rna.any():
        seq = np.where(np.repeat(rna, np.diff(seq_off)) & (seq == ord('U')), ord('T'), seq).astype(np.uint8)
    return np.ascontiguousarray(seq), rna


def parse_reads(data):
    """FASTQ or FASTA by the first character of the data, like get_sequence_file_type (misc.py:84-106).
    Returns (FastqBatch, 'fastq' | 'fasta')."""
    head = bytes(data[:1])
    if head == b'>':
        return parse_fasta(data), 'fasta'
    if head in (b'@', b''):
        return parse_fastq(data), 'fastq'
    raise ValueError('File is neither FASTA or FASTQ')


def _parse_fastq_native(buf):
    """parse_fastq through libhostio.so (include/porechop_b200_io.h): index the records, then parallel memcpy."""
    name_a, name_len, seq_a, seq_len, qual_a, qual_len = hostio.fastq_index(buf)
    name_buf, name_off = hostio.gather(buf, name_a, name_len)
    seq, seq_off = hostio.gather(buf, seq_a, seq_len)
    rna = hostio.normalise(seq, seq_off)
    qual, qual_off = hostio.gather(buf, qual_a, np.maximum(qual_len, seq_len), src_len=qual_len, fill=ord('+'))
    return FastqBatch(name_buf, name_off, seq, seq_off, qual, qual_off, rna)


def _segment_sums(flags, off):
    c = np.zeros(len(flags) + 1, dtype=np.int64)
    np.cumsum(flags, out=c[1:])
    return c[off[1:]] - c[off[:-1]]


def _pad_segments(buf, off, pad, fill):
    lens = np.diff(off) + pad
    new_off = np.zeros(len(off), dtype=np.int64)
    np.cumsum(lens, out=new_off[1:])
    out = np.full(int(new_off[-1]), fill, dtype=np.uint8)
    _scatter(out, new_off[:-1], buf, off[:-1], np.diff(off))
    return out, new_off


def _ramp(lens):
    """concatenated arange(l) for l in lens, plus the segment id of every element."""
    lens = np.asarray(lens, dtype=np.int64)
    total = int(lens.sum())
    first = np.zeros(len(lens), dtype=np.int64)
    np.cumsum(lens[:-1], out=first[1:])
    seg = np.repeat(np.arange(len(lens), dtype=np.int64), lens)
    return np.arange(total, dtype=np.int64) - first[seg], seg


def _gather_ranges(buf, a, b, alloc=None):
    """concatenate buf[a[i]:b[i]] for all i -> (flat uint8, int64 offsets) without a Python loop.
    alloc: optional allocator of the flat result (hostio.gather)."""
    lens = np.maximum(np.asarray(b, dtype=np.int64) - np.asarray(a, dtype=np.int64), 0)
    if hostio.LIB is not None and buf.dtype == np.uint8 and buf.flags.c_contiguous:
        return hostio.gather(buf, a, lens, alloc=alloc)
    off = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    if int(off[-1]) == 0:
        return np.zeros(0, dtype=np.uint8), off
    k, seg = _ramp(lens)
    return np.ascontiguousarray(buf[np.asarray(a, dtype=np.int64)[seg] + k]), off


def _scatter(out, dst_start, src, src_start, lens):
    """out[dst_start[i] + k] = src[src_start[i] + k] for k < lens[i]."""
    if len(lens) == 0 or int(np.sum(lens)) == 0:
        return
    k, seg = _ramp(lens)
    out[np.asarray(dst_start, dtype=np.int64)[seg] + k] = src[np.asarray(src_start, dtype=np.int64)[seg] + k]


# ---------------------------------------------------------------------------------------------------------------
def end_windows(seq, seq_off, end_size):
    """(start windows, end windows) as two ragged batches (buf, off): window length = min(end_size, read length),
    exactly `seq[:end_size]` and `seq[-end_size:]` of nanopore_read.py:172,194."""
    lens = np.diff(seq_off)
    wl = np.minimum(lens, end_size).astype(np.int64)
    start = _gather_ranges(seq, seq_off[:-1], seq_off[:-1] + wl)
    end = _gather_ranges(seq, seq_off[1:] - wl, seq_off[1:])
    return start, end


def end_trim_amounts(start_records, end_records, end_size, extra_trim_size, end_threshold, min_trim_size):
    """The trim rule of find_start_trim / find_end_trim (nanopore_read.py:178-180, 200-202) on record arrays of
    shape [n_reads, n_adapters, 9].  Returns (start_trim[n], end_trim[n]) -- the max over the adapters that pass."""
    def one(rec, is_start):
        n, a = rec.shape[0], rec.shape[1]
        if a == 0 or n == 0:
            return np.zeros(n, dtype=np.int64)
        if hostio.LIB is not None:                    # one parallel pass in C (libhostio.so), same rule
            return hostio.end_trim(rec, is_start, end_size, extra_trim_size, end_threshold, min_trim_size)
        _, part, rs, re_ = scores_from_records(rec.reshape(-1, 9))
        part, rs, re_ = part.reshape(n, a), rs.reshape(n, a), re_.reshape(n, a)
        with np.errstate(invalid='ignore'):
            ok = (part > end_threshold) & ((re_ - rs) >= min_trim_size)
        if is_start:
            ok &= re_ != end_size
            amount = re_ + extra_trim_size
        else:
            ok &= rs != 0
            amount = (end_size - rs) + extra_trim_size
        return np.where(ok, amount, 0).max(axis=1)
    return one(np.asarray(start_records), True), one(np.asarray(end_records), False)


# Decisions on the device (SURVEY 8(f) row 3, include/porechop_b200.h adapterEndDecisions): the engine reduces the records
# of the end windows to per-read trim amounts + the barcode score pairs before anything is copied back.  Off by default.
DEVICE_DECISIONS = os.environ.get('PB200_DEVICE_DECISIONS', '0') == '1'


class PairScores:
    """Barcode score columns as the device returns them: (match_ad, len_ad) uint16 pairs for the requested adapter
    columns.  full(cols) gives the same doubles as the record path (float("%f" % (100.0 * match / len)))."""

    def __init__(self, cols, pairs):
        self.cols = [int(c) for c in cols]
        self.pairs = pairs                            # uint16[n, len(cols), 2]

    def full(self, cols):
        assert [int(c) for c in cols] == self.cols
        if self.pairs.shape[1] == 0:
            return np.zeros((self.pairs.shape[0], 0))
        from .align import _percent_exact
        return _percent_exact(self.pairs[:, :, 0], self.pairs[:, :, 1])


def trim_end_adapters(batch, start_adapters, end_adapters, scoring_scheme_vals, end_size=150, extra_trim_size=2,
                      end_threshold=75.0, min_trim_size=4, device_decisions=None, score_cols=None, rank_names=None):
    """Phase B for a FastqBatch and fixed adapter lists (sequences): returns (start_trim, end_trim, start_records,
    end_records).  Two batched engine calls, no per-read Python.
    device_decisions (default: the module switch DEVICE_DECISIONS): one adapterEndDecisions submit instead -- the trim
    rule runs on the device and the last two results are PairScores for score_cols = (start columns, end columns) -- or, with
    rank_names = (start names, end names) (one unique barcode name per score column), Top2Scores: the barcode ranking of
    determine_barcode is done on the device as well and 24 bytes per window come back instead of 4 per score column."""
    (sbuf, soff), (ebuf, eoff) = end_windows(batch.seq, batch.seq_off, end_size)
    n = len(batch)
    if device_decisions is None:
        device_decisions = DEVICE_DECISIONS
    if device_decisions and n > 0 and end_threshold >= 0 and (start_adapters or end_adapters):
        scols, ecols = score_cols if score_cols is not None else ((), ())
        sa, so = W.pack_sequences(start_adapters, offset_dtype=np.int32)
        ea, eo = W.pack_sequences(end_adapters, offset_dtype=np.int32)
        (st, sp, _), (et, ep, _) = W.adapter_end_decisions(
            [(sbuf, soff, sa, so, True, list(scols)), (ebuf, eoff, ea, eo, False, list(ecols))], scoring_scheme_vals,
            end_size, extra_trim_size, end_threshold, min_trim_size, want_top2=rank_names is not None)
        if rank_names is not None:
            return st.astype(np.int64), et.astype(np.int64), Top2Scores(rank_names[0], sp), Top2Scores(rank_names[1], ep)
        return st.astype(np.int64), et.astype(np.int64), PairScores(scols, sp), PairScores(ecols, ep)

    def run(buf, off, adapters):
        if not adapters or n == 0:
            return np.zeros((n, 0, 9), dtype=np.int32)
        abuf, aoff = W.pack_sequences(adapters, offset_dtype=np.int32)
        return W.adapter_alignment_batch(buf, off, abuf, aoff, scoring_scheme_vals).reshape(n, len(adapters), 9)
    srec, erec = run(sbuf, soff, start_adapters), run(ebuf, eoff, end_adapters)
    st, et = end_trim_amounts(srec, erec, end_size, extra_trim_size, end_threshold, min_trim_size)
    return st, et, srec, erec


# ---------------------------------------------------------------------------------------------------------------
def trimmed_ranges(lens, start_trim, end_trim):
    """[a, b) of `x[start_trim : len(x) - end_trim]` for every read, with Python's slice semantics
    (nanopore_read.py:57-63): an end position that goes negative (end trim larger than a short read) counts from the
    END of the read again -- the reference's behaviour, reproduced on purpose.  Untrimmed reads keep [0, len)."""
    lens = np.asarray(lens, dtype=np.int64)
    st, et = np.asarray(start_trim, dtype=np.int64), np.asarray(end_trim, dtype=np.int64)
    e = lens - et
    e = np.where(e < 0, np.maximum(e + lens, 0), e)
    a = np.minimum(st, lens)
    b = np.maximum(np.minimum(e, lens), a)
    untouched = (st == 0) & (et == 0)
    return np.where(untouched, 0, a), np.where(untouched, lens, b)


# The whole middle scan on the device (include/porechop_b200.h adapterMiddleScan): masking rounds included, one engine call,
# the masked reads and the records of reads without a hit stay on the device.  Off by default.
DEVICE_MIDDLE = os.environ.get('PB200_DEVICE_MIDDLE', '0') == '1'


def find_middle_hits(batch, start_trim, end_trim, adapters, middle_threshold, scoring_scheme_vals, device=None):
    """Phase C.  adapters: list of (name, sequence) in the reference's order (porechop.py:541-548).
    Returns {read index: [(adapter position, read_start, read_end, full_score), ...]} in the order the reference finds
    them; coordinates are in the trimmed read.  Round 0 is one cross product over all trimmed reads; only reads with
    a hit are masked with '-' and re-submitted (as a pair list) from the adapter that hit.
    device (default: the module switch DEVICE_MIDDLE): one adapterMiddleScan call runs every round on the device instead;
    the same dict comes back.  Inputs the device scan does not take (threshold <= 0, adapters with other bases than
    A/C/G/T/U, scoring schemes outside the int16 kernels: PB200_ERR_ARG) use the rounds above."""
    n, n_ad = len(batch), len(adapters)
    hits = {}
    if n == 0 or n_ad == 0:
        return hits
    if device is None:
        device = DEVICE_MIDDLE
    a, b = trimmed_ranges(batch.lengths(), start_trim, end_trim)
    # the trimmed reads of the chunk go into the engine's pinned staging buffer (reused chunk after chunk, uploaded by DMA at
    # PCIe speed) when there is one: a gather into fresh pageable memory + its upload would take far longer than the device
    pinned = getattr(W, 'pinned_buffer', None)
    tbuf, toff = _gather_ranges(batch.seq, batch.seq_off[:-1] + a, batch.seq_off[:-1] + b,
                                alloc=(lambda nbytes: pinned(0, nbytes)) if pinned is not None else None)
    abuf, aoff = W.pack_sequences([x[1] for x in adapters], offset_dtype=np.int32)
    if device:
        try:
            n_hits, h = W.adapter_middle_scan(tbuf, toff, abuf, aoff, scoring_scheme_vals, middle_threshold)
        except W.EngineError as e:
            if e.code != W.ERR_ARG:
                raise
        else:
            return _hits_dict(n_hits, h)
    rec = W.adapter_alignment_batch(tbuf, toff, abuf, aoff, scoring_scheme_vals)
    full, _, rs, re_ = (x.reshape(n, n_ad) for x in scores_from_records(rec))
    hit = full >= middle_threshold                           # NaN never hits, as in the reference
    first = hit.argmax(axis=1)
    active = []                                              # [read, masked bytearray, adapter position]
    for i in np.flatnonzero(hit.any(axis=1)):
        p = int(first[i])
        x, y = int(rs[i, p]), int(re_[i, p])
        masked = bytearray(tbuf[toff[i]:toff[i + 1]].tobytes())
        masked[x:y] = b'-' * (y - x)
        hits[int(i)] = [(p, x, y, float(full[i, p]))]
        active.append([int(i), masked, p])
    while active:
        sbuf, soff = W.pack_sequences([bytes(m) for _, m, _ in active], offset_dtype=np.int64)
        ps = np.concatenate([np.full(n_ad - p, k, dtype=np.int32) for k, (_, _, p) in enumerate(active)])
        pa = np.concatenate([np.arange(p, n_ad, dtype=np.int32) for _, _, p in active])
        rec = W.adapter_alignment_batch(sbuf, soff, abuf, aoff, scoring_scheme_vals, ps, pa)
        full, _, rs, re_ = scores_from_records(rec)
        base, still = 0, []
        for i, masked, p in active:
            cnt = n_ad - p
            h = np.flatnonzero(full[base:base + cnt] >= middle_threshold)
            if len(h):
                q = base + int(h[0])
                x, y = int(rs[q]), int(re_[q])
                masked[x:y] = b'-' * (y - x)
                hits[i].append((p + int(h[0]), x, y, float(full[q])))
                still.append([i, masked, p + int(h[0])])
            base += cnt
        active = still
    return hits


def _hits_dict(n_hits, h):
    """n_hits / hits of adapterMiddleScan (or adapterTrimReads) -> the dict find_middle_hits returns"""
    hits = {}
    full, _, rs, re_ = scores_from_records(np.ascontiguousarray(h[:, 1:]))
    reads = np.repeat(np.arange(len(n_hits)), n_hits)
    for k in range(len(h)):
        hits.setdefault(int(reads[k]), []).append((int(h[k, 0]), int(rs[k]), int(re_[k]), float(full[k])))
    return hits


def middle_trim_ranges(hits, adapters, start_sequence_names, end_sequence_names, extra_middle_trim_good_side=10,
                       extra_middle_trim_bad_side=100):
    """hits of find_middle_hits -> {read index: [(trim_start, trim_end), ...]}: the ranges the reference adds to
    `middle_trim_positions` (nanopore_read.py:231-240), in trimmed-read coordinates (may stick out of the read)."""
    out = {}
    for i, hs in hits.items():
        r = []
        for p, x, y, _ in hs:
            name = adapters[p][0]
            r.append((x - (extra_middle_trim_bad_side if name in start_sequence_names else extra_middle_trim_good_side),
                      y + (extra_middle_trim_bad_side if name in end_sequence_names else extra_middle_trim_good_side)))
        out[i] = r
    return out


# ---------------------------------------------------------------------------------------------------------------
def _numbered_name(name, number):
    # add_number_to_read_name (nanopore_read.py:494-498)
    tag = b'_' + str(number).encode()
    return name + tag if b' ' not in name else name.replace(b' ', tag + b' ', 1)


def _split_parts(length, ranges, min_split_read_size):
    """runs of positions of [0, length) outside every range, at least min_split_read_size long
    (get_split_read_parts, nanopore_read.py:76-95)."""
    keep = np.ones(length, dtype=bool)
    for x, y in ranges:
        x, y = max(x, 0), min(y, length)
        if y > x:
            keep[x:y] = False
    edge = np.flatnonzero(np.diff(np.concatenate([[0], keep.view(np.int8), [0]])))
    return [(int(s), int(e)) for s, e in zip(edge[0::2], edge[1::2]) if e - s >= min_split_read_size]


def emit(batch, start_trim=None, end_trim=None, middle=None, fmt='fastq', min_split_read_size=1000,
         discard_middle=False, untrimmed=False, select=None, chunk_bytes=64 << 20, as_array=False):
    """What the reference writes for these reads, in read order, as bytes: get_fastq / get_fasta of every read
    (nanopore_read.py:97-147).  middle: {read index: [(trim_start, trim_end), ...]} from middle_trim_ranges -- a read
    listed there is split (or dropped with discard_middle); `select` (bool[n]) keeps a subset (e.g. one barcode bin).
    Reads whose trimmed sequence is empty are not written.  fmt: 'fastq' or 'fasta' (70 columns, misc.py:327-338).
    as_array=True returns the uint8 array the C writer filled (file.write() takes it as is) instead of copying it
    into a bytes object."""
    n = len(batch)
    lens = batch.lengths()
    z = np.zeros(n, dtype=np.int64)
    st = z if start_trim is None else np.asarray(start_trim, dtype=np.int64)
    et = z if end_trim is None else np.asarray(end_trim, dtype=np.int64)
    a, b = trimmed_ranges(lens, st, et)
    qlens = np.diff(batch.qual_off)
    qa, qb = trimmed_ranges(qlens, st, et)
    middle = middle or {}
    plain = np.ones(n, dtype=bool)
    if middle:
        plain[np.fromiter(middle.keys(), dtype=np.int64, count=len(middle))] = False
    if select is not None:
        plain &= np.asarray(select, dtype=bool)
    # ---- output records: (read, seq [s0, s1), first quality, name [n0, n1) in `names`) ----
    names, name_off = batch.name_buf, batch.name_off
    idx = np.flatnonzero(plain)
    if untrimmed:
        r_s0, r_s1, r_q0, r_ql = z[idx], lens[idx], z[idx], qlens[idx]
    else:
        r_s0, r_s1, r_q0, r_ql = a[idx], b[idx], qa[idx], (qb - qa)[idx]
    r_read, r_n0, r_n1 = idx, name_off[idx], name_off[idx + 1]
    order_key = idx.astype(np.float64)
    if middle and not discard_middle:
        x_read, x_s0, x_s1, x_q0, x_name, x_key = [], [], [], [], [], []
        nb = names.tobytes()
        for i in sorted(middle):
            if select is not None and not select[i]:
                continue
            nm = nb[name_off[i]:name_off[i + 1]]
            parts = _split_parts(int(b[i] - a[i]), middle[i], min_split_read_size)
            for k, (s, e) in enumerate(parts):
                x_read.append(i)
                x_s0.append(int(a[i]) + s)
                x_s1.append(int(a[i]) + e)
                x_q0.append(int(qa[i]) + s)
                x_name.append(_numbered_name(nm, k + 1))
                x_key.append(i + (k + 1) / (len(parts) + 1.0))
        if x_read:
            extra, extra_off = W.pack_sequences(x_name, offset_dtype=np.int64)
            base = len(names)
            names = np.concatenate([names, extra])
            r_read = np.concatenate([r_read, np.array(x_read, dtype=np.int64)])
            r_s0 = np.concatenate([r_s0, np.array(x_s0, dtype=np.int64)])
            r_s1 = np.concatenate([r_s1, np.array(x_s1, dtype=np.int64)])
            r_q0 = np.concatenate([r_q0, np.array(x_q0, dtype=np.int64)])
            r_ql = np.concatenate([r_ql, np.array(x_s1, dtype=np.int64) - np.array(x_s0, dtype=np.int64)])
            r_n0 = np.concatenate([r_n0, base + extra_off[:-1]])
            r_n1 = np.concatenate([r_n1, base + extra_off[1:]])
            order_key = np.concatenate([order_key, np.array(x_key)])
    keep = r_s1 > r_s0                                        # "Don't return empty sequences"
    o = np.argsort(order_key[keep], kind='stable')
    r_read, r_s0, r_s1, r_q0, r_ql, r_n0, r_n1 = (v[keep][o] for v in (r_read, r_s0, r_s1, r_q0, r_ql, r_n0, r_n1))
    # ---- assemble, a bounded number of output bytes at a time ----
    slen, nlen = r_s1 - r_s0, r_n1 - r_n0
    if fmt == 'fastq':
        rec_len = 1 + nlen + 1 + slen + 3 + r_ql + 1
    elif fmt == 'fasta':
        rec_len = 1 + nlen + 1 + slen + (slen + 69) // 70
    else:
        raise ValueError("fmt must be 'fastq' or 'fasta'")
    if hostio.LIB is not None:
        out_off = np.zeros(len(rec_len) + 1, dtype=np.int64)
        np.cumsum(rec_len, out=out_off[1:])
        out = hostio.emit(out_off, fmt, np.ascontiguousarray(names), r_n0, nlen, batch.seq, batch.seq_off[r_read] + r_s0, slen,
                          batch.qual, batch.qual_off[r_read] + r_q0, r_ql, batch.rna[r_read])
        return out if as_array else out.tobytes()
    pieces, lo = [], 0
    csum = np.cumsum(rec_len)
    while lo < len(rec_len):
        hi = int(np.searchsorted(csum, (csum[lo - 1] if lo else 0) + chunk_bytes, side='right'))
        hi = max(hi, lo + 1)
        sl = slice(lo, hi)
        pieces.append(_assemble(batch, names, fmt, r_read[sl], r_s0[sl], slen[sl], r_q0[sl], r_ql[sl], r_n0[sl], nlen[sl],
                                rec_len[sl]))
        lo = hi
    out = b''.join(pieces)
    return np.frombuffer(out, dtype=np.uint8) if as_array else out


def _assemble(batch, names, fmt, read, s0, slen, q0, qlen, n0, nlen, rec_len):
    off = np.zeros(len(rec_len) + 1, dtype=np.int64)
    np.cumsum(rec_len, out=off[1:])
    out = np.full(int(off[-1]), 10, dtype=np.uint8)              # every byte not written below is a '\n'
    p = off[:-1]
    out[p] = ord('@') if fmt == 'fastq' else ord('>')
    _scatter(out, p + 1, names, n0, nlen)
    sp = p + 1 + nlen + 1                                       # first base
    src0 = batch.seq_off[read] + s0
    k, seg = _ramp(slen)
    vals = batch.seq[src0[seg] + k]
    if batch.rna[read].any():                                   # RNA reads go back out as U (nanopore_read.py:107,133)
        vals = np.where(batch.rna[read][seg] & (vals == ord('T')), ord('U'), vals).astype(np.uint8)
    if fmt == 'fastq':
        out[sp[seg] + k] = vals
        out[sp + slen + 1] = ord('+')
        _scatter(out, sp + slen + 3, batch.qual, batch.qual_off[read] + q0, qlen)
    else:
        out[sp[seg] + k + k // 70] = vals                       # a '\n' after every 70 bases and after the last one
    return out.tobytes()


# ---------------------------------------------------------------------------------------------------------------
# Phase A on the device (include/porechop_b200.h adapterSetSearch): the records of the search are reduced to one best score
# per adapter sequence before anything is copied back -- 8 bytes per sequence instead of 36 per (window, sequence).  Off by
# default.
DEVICE_SEARCH = os.environ.get('PB200_DEVICE_SEARCH', '0') == '1'


def search_adapter_sets(batch, adapter_sets, scoring_scheme_vals, check_reads=10000, end_size=150, device=None):
    """Phase A (porechop.py:286-327, nanopore_read.py:149-164) on a FastqBatch: the best full-adapter identity of every
    set's start / end sequence over the end windows of the first `check_reads` reads.  adapter_sets as for trim_fastq.
    Returns (best_start_score[k], best_end_score[k]) (0.0 where a set has no such sequence); the caller applies the
    reference's policy on top (`>= adapter_threshold`, porechop.py:327; 1D^2 fix-up, barcode kit choice).
    device (default: the module switch DEVICE_SEARCH): one adapterSetSearch call with both batches instead; the same
    scores come back."""
    if device is None:
        device = DEVICE_SEARCH
    sets = _norm_sets(adapter_sets)
    k = min(int(check_reads), len(batch))
    best_s, best_e = np.zeros(len(sets)), np.zeros(len(sets))
    if k == 0:
        return best_s, best_e
    (sbuf, soff), (ebuf, eoff) = end_windows(batch.seq, batch.seq_off[:k + 1], end_size)
    searched = []
    for which, buf, off, best in ((1, sbuf, soff, best_s), (2, ebuf, eoff, best_e)):
        idx = [j for j, t in enumerate(sets) if t[which]]
        if not idx:
            continue
        abuf, aoff = W.pack_sequences([sets[j][which][1] for j in idx], offset_dtype=np.int32)
        if device:
            searched.append((idx, best, (buf, off, abuf, aoff)))
            continue
        rec = W.adapter_alignment_batch(buf, off, abuf, aoff, scoring_scheme_vals)
        full, _, _, _ = scores_from_records(rec)
        best[idx] = np.maximum(full.reshape(k, len(idx)).max(axis=0), 0.0)
    if searched:
        for (idx, best, _), got in zip(searched, W.adapter_set_search([x[2] for x in searched], scoring_scheme_vals)):
            best[idx] = got
    return best_s, best_e


def _norm_sets(matching_sets):
    """adapter sets as (name, start, end) with start / end = (name, sequence) or None; (start, end) pairs get name ''."""
    out = []
    for t in matching_sets:
        name, s, e = t if len(t) == 3 else ('', t[0], t[1])
        out.append((name, tuple(s) if s else None, tuple(e) if e else None))
    return out


def _middle_adapters(sets):
    adapters = []
    for _, s, e in sets:                                        # porechop.py:541-548
        if s:
            adapters.append(s)
        if e and ((not s) or e[1] != s[1]):
            adapters.append(e)
    return adapters


def _trim_reads_fused(batch, starts, ends, adapters, scoring_scheme_vals, end_size, extra_end_trim, end_threshold,
                      min_trim_size, middle_threshold, score_cols, rank_names):
    """Phase B + Phase C in one adapterTrimReads call: the reads go up once, and the trims, the score outputs and the hits come
    back.  Returns what trim_end_adapters (device decisions) and find_middle_hits (device scan) return together, or None when
    the engine does not take these inputs (PB200_ERR_ARG): the caller then runs the two calls."""
    scols, ecols = score_cols if score_cols is not None else ((), ())
    sa, so = W.pack_sequences(starts, offset_dtype=np.int32)
    ea, eo = W.pack_sequences(ends, offset_dtype=np.int32)
    middle = W.pack_sequences([x[1] for x in adapters], offset_dtype=np.int32) if adapters else None
    seq = batch.seq
    pinned = getattr(W, 'pinned_buffer', None)
    if pinned is not None and hostio.LIB is not None and len(seq):
        # the bases go up from the engine's pinned staging buffer (DMA at PCIe speed): the upload of a pageable batch is staged
        # by the driver and took longer than this parallel copy (64 KB pieces for the copy's thread team) plus the DMA
        piece = 1 << 16
        a = np.arange(0, len(seq), piece, dtype=np.int64)
        seq, _ = hostio.gather(seq, a, np.minimum(piece, len(seq) - a), alloc=lambda nbytes: pinned(0, nbytes))
    try:
        st, et, sp, ep, n_hits, h = W.adapter_trim_reads(
            seq, batch.seq_off, (sa, so, list(scols)), (ea, eo, list(ecols)), middle, scoring_scheme_vals, end_size,
            extra_end_trim, end_threshold, min_trim_size, middle_threshold, want_top2=rank_names is not None)
    except W.EngineError as e:
        if e.code != W.ERR_ARG:
            raise
        return None
    if rank_names is not None:
        srec, erec = Top2Scores(rank_names[0], sp), Top2Scores(rank_names[1], ep)
    else:
        srec, erec = PairScores(scols, sp), PairScores(ecols, ep)
    return st.astype(np.int64), et.astype(np.int64), srec, erec, _hits_dict(n_hits, h)


def _run_trim(data, matching_sets, scoring_scheme_vals, end_size, extra_end_trim, end_threshold, min_trim_size, no_split,
              middle_threshold, good_side, bad_side, score_cols=None, rank_names=None, device_trim=None):
    """device_trim (default: both DEVICE_DECISIONS and DEVICE_MIDDLE): Phase B and Phase C in one adapterTrimReads call
    instead of adapterEndDecisions + adapterMiddleScan; inputs that call does not take run the two calls."""
    t0 = time.perf_counter()
    batch = data if isinstance(data, FastqBatch) else parse_fastq(data)
    t1 = time.perf_counter()
    sets = _norm_sets(matching_sets)
    starts = [s[1] for _, s, _ in sets if s]
    ends = [e[1] for _, _, e in sets if e]
    adapters = [] if no_split else _middle_adapters(sets)
    if device_trim is None:
        device_trim = DEVICE_DECISIONS and DEVICE_MIDDLE
    fused = None
    if device_trim and len(batch) > 0 and end_threshold >= 0 and (starts or ends):
        fused = _trim_reads_fused(batch, starts, ends, adapters, scoring_scheme_vals, end_size, extra_end_trim, end_threshold,
                                  min_trim_size, middle_threshold, score_cols, rank_names)
    if fused is not None:
        st, et, srec, erec, hits = fused
        t2 = time.perf_counter()
    else:
        st, et, srec, erec = trim_end_adapters(batch, starts, ends, scoring_scheme_vals, end_size, extra_end_trim,
                                               end_threshold, min_trim_size, score_cols=score_cols, rank_names=rank_names)
        t2 = time.perf_counter()
        hits = {} if no_split else find_middle_hits(batch, st, et, adapters, middle_threshold, scoring_scheme_vals)
    middle = {}
    if not no_split:
        middle = middle_trim_ranges(hits, adapters, {s[0] for _, s, _ in sets if s}, {e[0] for _, _, e in sets if e},
                                    good_side, bad_side)
    seconds = {'parse': t1 - t0, 'end_trim': t2 - t1, 'middle': time.perf_counter() - t2}
    return batch, sets, st, et, srec, erec, middle, seconds


def trim_fastq(data, matching_sets, scoring_scheme_vals, end_size=150, extra_end_trim=2, end_threshold=75.0,
               min_trim_size=4, no_split=False, middle_threshold=85.0, extra_middle_trim_good_side=10,
               extra_middle_trim_bad_side=100, min_split_read_size=1000, discard_middle=False, fmt='fastq', as_array=False,
               device_trim=None):
    """FASTQ bytes -> the bytes `porechop -i in.fastq -o out.<fmt>` writes once Phase A has chosen `matching_sets`
    (porechop.py:54-79).  matching_sets: list of (start, end) with start / end = (name, sequence) or None -- the
    `start_sequence` / `end_sequence` of the reference's Adapter objects (adapters.py:18-30).
    device_trim: see _run_trim (default: one adapterTrimReads call when DEVICE_DECISIONS and DEVICE_MIDDLE are both on).
    Returns (output bytes, info dict with the per-read decisions)."""
    batch, _, st, et, _, _, middle, seconds = _run_trim(data, matching_sets, scoring_scheme_vals, end_size, extra_end_trim,
                                                        end_threshold, min_trim_size, no_split, middle_threshold,
                                                        extra_middle_trim_good_side, extra_middle_trim_bad_side,
                                                        device_trim=device_trim)
    t0 = time.perf_counter()
    out = emit(batch, st, et, middle, fmt, min_split_read_size, discard_middle, as_array=as_array)
    seconds['emit'] = time.perf_counter() - t0
    return out, {'start_trim': st, 'end_trim': et, 'middle': middle, 'n_reads': len(batch), 'seconds': seconds}


# ---------------------------------------------------------------------------------------------------------------
def _barcode_name(name, start, end):
    # Adapter.get_barcode_name (adapters.py:40-52): the shortest of the set / start / end names (first on ties)
    names = [name] + ([start[0]] if start else []) + ([end[0]] if end else [])
    return sorted(names, key=len)[0].replace(' ', '_')


def _dict_columns(names):
    """the reference keeps barcode scores in a dict keyed by barcode name (nanopore_read.py:181-183): a repeated name
    keeps its FIRST position and its LAST value.  Returns (unique names in insertion order, column holding the value)."""
    last = {}
    for j, nm in enumerate(names):
        last[nm] = j
    return list(last.keys()), [last[nm] for nm in last]


def call_barcodes(start_scores, start_names, end_scores, end_names, barcode_threshold=75.0, barcode_diff=5.0,
                  require_two_barcodes=False, albacore_calls=None):
    """determine_barcode (nanopore_read.py:399-470) for all reads at once.  start_scores: float[n, len(start_names)]
    = full-adapter identity of every read's start window against the barcode start sequences, columns in adapter
    order (ties go to the earlier column, as Python's stable reverse sort does); same for the end.  Returns a list of
    barcode names ('none' = unclassified)."""
    start_scores, end_scores = np.asarray(start_scores, dtype=np.float64), np.asarray(end_scores, dtype=np.float64)
    n = start_scores.shape[0] if start_scores.ndim == 2 else end_scores.shape[0]
    s_names, s_cols = _dict_columns(start_names)
    e_names, e_cols = _dict_columns(end_names)
    S = start_scores[:, s_cols] if s_cols else np.zeros((n, 0))
    E = end_scores[:, e_cols] if e_cols else np.zeros((n, 0))

    def best_two(M, ids):
        """(best column, best score, second score) per row; second = best score among columns with another id."""
        if M.shape[1] == 0:
            return np.full(n, -1), np.zeros(n), np.zeros(n)
        bcol = M.argmax(axis=1)
        bscore = M[np.arange(n), bcol]
        other = np.where(ids[None, :] == ids[bcol][:, None], -np.inf, M)
        sscore = other.max(axis=1) if M.shape[1] > 1 else np.full(n, -np.inf)
        return bcol, bscore, np.where(np.isfinite(sscore), sscore, 0.0)      # ('none', 0.0) when there is no second

    if require_two_barcodes:
        sc, sb, ss = best_two(S, np.arange(len(s_names)))
        ec, eb, es = best_two(E, np.arange(len(e_names)))
        sn = np.array(s_names + ['none'], dtype=object)[sc]
        en = np.array(e_names + ['none'], dtype=object)[ec]
        ok = (sb >= barcode_threshold) & (eb >= barcode_threshold) & (sb >= ss + barcode_diff) & \
             (eb >= es + barcode_diff) & (sn == en)
        calls = np.where(ok, sn, 'none')
    else:
        all_names = list(dict.fromkeys(s_names + e_names))
        ids = np.array([all_names.index(nm) for nm in s_names + e_names], dtype=np.int64)
        C = np.concatenate([S, E], axis=1)
        bc, bb, bs = best_two(C, ids)
        best_id = ids[bc] if len(ids) else np.full(n, -1)           # -1 -> 'none' (no barcode column at all)
        bn = np.array(all_names + ['none'], dtype=object)[best_id]
        ok = (bb >= barcode_threshold) & (bb >= bs + barcode_diff)
        calls = np.where(ok, bn, 'none')
    calls = [str(c) for c in calls]
    if albacore_calls is not None:                            # Porechop and Albacore must agree (nanopore_read.py:466-470)
        calls = [c if (a is None or a == c) else 'none' for c, a in zip(calls, albacore_calls)]
    return calls


class Top2Scores:
    """Barcode ranking as the device returns it (adapterEndDecisions, `top2`): per read the (position, match_ad, len_ad) of the
    best and the second-best score column -- positions index `names` (every barcode name once, in score-column order)."""

    def __init__(self, names, top2):
        self.names = list(names)
        self.top2 = np.asarray(top2, dtype=np.int32).reshape(-1, 6)

    def ranked(self):
        """(pos1, score1, pos2, score2): positions (-1 = none) and the exact doubles the reference parses (0.0 for none)."""
        from .align import _percent_exact
        t = self.top2
        s1 = np.where(t[:, 0] >= 0, _percent_exact(t[:, 1], np.maximum(t[:, 2], 1)), 0.0)
        s2 = np.where(t[:, 3] >= 0, _percent_exact(t[:, 4], np.maximum(t[:, 5], 1)), 0.0)
        return t[:, 0].astype(np.int64), s1, t[:, 3].astype(np.int64), s2


def top2_from_scores(scores):
    """Host statement of the device ranking (tests, and the record path when only the ranking is wanted): float[n, k] ->
    (pos1, score1, pos2, score2) with ties going to the earlier column, -1 / 0.0 where there is no such column."""
    M = np.asarray(scores, dtype=np.float64)
    n, k = M.shape
    if k == 0:
        return np.full(n, -1), np.zeros(n), np.full(n, -1), np.zeros(n)
    order = np.argsort(-M, axis=1, kind='stable')
    p1 = order[:, 0]
    s1 = M[np.arange(n), p1]
    if k == 1:
        return p1, s1, np.full(n, -1), np.zeros(n)
    p2 = order[:, 1]
    return p1, s1, p2, M[np.arange(n), p2]


def call_barcodes_top2(start, end, barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=False,
                       albacore_calls=None):
    """determine_barcode (nanopore_read.py:399-470) from the per-side rankings alone: `start` / `end` are
    (unique names, (pos1, score1, pos2, score2)) -- Top2Scores.ranked() or top2_from_scores() over the dict-deduplicated
    columns.  A barcode name occurs at most once per side, so the best and second-best of the merged list
    (nanopore_read.py:441-456) are always among the two best of each side."""
    (s_names, (sp1, ss1, sp2, ss2)), (e_names, (ep1, es1, ep2, es2)) = start, end
    n = len(sp1)
    all_names = list(dict.fromkeys(list(s_names) + list(e_names)))
    idx = {nm: i for i, nm in enumerate(all_names)}
    none_id = len(all_names)
    name_arr = np.array(all_names + ['none'], dtype=object)
    s_ids = np.array([idx[nm] for nm in s_names] + [none_id], dtype=np.int64)     # position -1 -> 'none'
    e_ids = np.array([idx[nm] for nm in e_names] + [none_id], dtype=np.int64)
    sn1, sn2, en1, en2 = s_ids[sp1], s_ids[sp2], e_ids[ep1], e_ids[ep2]
    if require_two_barcodes:
        ok = (ss1 >= barcode_threshold) & (es1 >= barcode_threshold) & (ss1 >= ss2 + barcode_diff) & \
             (es1 >= es2 + barcode_diff) & (sn1 == en1)
        calls = np.where(ok, name_arr[sn1], 'none')
    else:
        have_s, have_e = sp1 >= 0, ep1 >= 0
        s_first = have_s & (~have_e | (ss1 >= es1))                    # stable sort: the start list comes first on ties
        best_id = np.where(s_first, sn1, np.where(have_e, en1, none_id))
        best = np.where(s_first, ss1, np.where(have_e, es1, 0.0))
        # best entry of each side whose name differs from the winner's (its first or its second entry)
        s_other = np.where(have_s & (sn1 != best_id), ss1, np.where((sp2 >= 0) & (sn2 != best_id), ss2, -np.inf))
        e_other = np.where(have_e & (en1 != best_id), es1, np.where((ep2 >= 0) & (en2 != best_id), es2, -np.inf))
        second = np.maximum(s_other, e_other)
        second = np.where(np.isfinite(second), second, 0.0)
        ok = (best >= barcode_threshold) & (best >= second + barcode_diff)
        calls = np.where(ok, name_arr[best_id], 'none')
    calls = [str(c) for c in calls]
    if albacore_calls is not None:
        calls = [c if (a is None or a == c) else 'none' for c, a in zip(calls, albacore_calls)]
    return calls if n else []


def demux_fastq(data, matching_sets, scoring_scheme_vals, forward_or_reverse='forward', end_size=150, extra_end_trim=2,
                end_threshold=75.0, min_trim_size=4, no_split=False, middle_threshold=85.0,
                extra_middle_trim_good_side=10, extra_middle_trim_bad_side=100, min_split_read_size=1000,
                discard_middle=False, barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=False,
                discard_unassigned=False, untrimmed=False, fmt='fastq', albacore_calls=None, as_array=False):
    """FASTQ bytes -> {bin name: bytes}: what `porechop -i in.fastq -b dir` writes into dir/<bin>.<fmt>
    (porechop.py:54-79, 652-676) once Phase A has chosen `matching_sets` = [(set name, start, end), ...] and the
    barcode direction.  A set is a barcode if its name starts with 'Barcode ' (adapters.py:31-32); its direction is
    'reverse' if its start name contains '_rev' (adapters.py:34-38).  Returns (bins, info)."""
    def is_bc(name, s):
        return name.startswith('Barcode ') and (('reverse' if '_rev' in s[0] else 'forward') == forward_or_reverse)
    sets = _norm_sets(matching_sets)
    s_sets = [t for t in sets if t[1]]
    e_sets = [t for t in sets if t[2]]
    s_cols = [j for j, (name, s, e) in enumerate(s_sets) if is_bc(name, s)]
    e_cols = [j for j, (name, s, e) in enumerate(e_sets) if is_bc(name, s)]
    s_names = [_barcode_name(*s_sets[j]) for j in s_cols]
    e_names = [_barcode_name(*e_sets[j]) for j in e_cols]
    # the reference's score dicts hold every barcode name once (first position, last value): rank exactly those columns
    (su, sk), (eu, ek) = _dict_columns(s_names), _dict_columns(e_names)
    s_cols, e_cols = [s_cols[k] for k in sk], [e_cols[k] for k in ek]
    batch, sets, st, et, srec, erec, middle, seconds = _run_trim(data, matching_sets, scoring_scheme_vals, end_size,
                                                                 extra_end_trim, end_threshold, min_trim_size, no_split,
                                                                 middle_threshold, extra_middle_trim_good_side,
                                                                 extra_middle_trim_bad_side, score_cols=(s_cols, e_cols),
                                                                 rank_names=(su, eu))
    t0 = time.perf_counter()
    n = len(batch)

    def full(rec, cols):
        if n == 0 or not cols:
            return np.zeros((n, len(cols)))
        if isinstance(rec, PairScores):               # decisions came from the device: only the score pairs exist
            return rec.full(cols)
        if hostio.LIB is not None:
            return hostio.full_scores(rec, cols)
        f, _, _, _ = scores_from_records(rec[:, cols, :].reshape(-1, 9))
        return f.reshape(n, len(cols))
    if isinstance(srec, Top2Scores):                  # the ranking came from the device too
        calls = call_barcodes_top2((su, srec.ranked()), (eu, erec.ranked()), barcode_threshold, barcode_diff,
                                   require_two_barcodes, albacore_calls)
    else:
        calls = call_barcodes(full(srec, s_cols), su, full(erec, e_cols), eu, barcode_threshold, barcode_diff,
                              require_two_barcodes, albacore_calls)
    calls_arr = np.array(calls, dtype=object)
    bins = {}
    for name in dict.fromkeys(calls):
        if discard_unassigned and name == 'none':
            continue
        out = emit(batch, st, et, middle, fmt, min_split_read_size, discard_middle, untrimmed, select=(calls_arr == name),
                   as_array=as_array)
        if len(out):
            bins[name] = out
    seconds['call_and_emit'] = time.perf_counter() - t0
    return bins, {'start_trim': st, 'end_trim': et, 'middle': middle, 'calls': calls, 'n_reads': n, 'seconds': seconds}
