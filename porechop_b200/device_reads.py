"""
Porechop on reads that are already in GPU memory: trimmed and split output reads, with their qualities, and the bytes of
Porechop's output files, in GPU memory.

For callers whose reads live on the device (a basecaller on the same card, a torch pipeline): one
adapterTrimSplitReadsDevice call runs Phase B (end trims), Phase C (middle adapters) and cuts the records Porechop writes --
the records fastq.emit would write for the same decisions, in the same order -- into device tensors.  Only the decisions
(trims, hits, barcode rankings) come to the host; the bases and qualities never do.  emit_reads (pb200EmitReadsDevice) then
formats the records on the device -- the bytes fastq.emit_parts writes: numbered names of split parts, U for RNA reads,
70-column FASTA -- so that the file's bytes come home in one copy:

    import torch
    from porechop_b200 import device_reads
    out = device_reads.trim_reads(seq, seq_off, matching_sets, (3, -6, -5, -2), qual)
    # out.seq / out.qual / out.off / out.read / out.part: CUDA tensors; record r is seq[off[r]:off[r+1]] of read read[r],
    # part[r] = 0 (not split) or k >= 1 (the k-th part).  names / name_off: the reads' names as CUDA tensors (uint8, int64).
    em = device_reads.emit_reads(out, names, name_off, rna, 'fastq')
    data = torch.empty(em.data.numel(), dtype=torch.uint8, pin_memory=True).copy_(em.data)
    open('out.fastq', 'wb').write(data.numpy())

demux_reads does the same for `porechop -b DIR`: it also calls every read's barcode on the device and returns the records
grouped by bin, so that each bin's reads are one contiguous slice of records and bytes:

    out = device_reads.demux_reads(seq, seq_off, matching_sets, (3, -6, -5, -2), qual, forward_or_reverse='forward',
                                   barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=False,
                                   discard_unassigned=False)
    em = device_reads.emit_reads(out, names, name_off, rna, 'fastq')
    data = torch.empty(em.data.numel(), dtype=torch.uint8, pin_memory=True).copy_(em.data)
    for name, (b0, b1) in em.bins.items():           # the bytes demux_fastq writes into <name>.fastq
        open(name + '.fastq', 'wb').write(data[b0:b1].numpy())

The device work runs on torch.cuda.current_stream(); the call returns when the outputs are written.  `W` (the engine's
wrapper module) and `device()` (the allocator) are module attributes, so that the same set handling and retry logic can run
on another engine build.
"""
import collections

import numpy as np

from . import cpp_function_wrappers as W
from . import fastq

TrimmedReads = collections.namedtuple('TrimmedReads', 'seq qual off read part start_trim end_trim hits calls')
DemuxedReads = collections.namedtuple('DemuxedReads', 'seq qual off read part bins calls start_trim end_trim hits')
EmittedReads = collections.namedtuple('EmittedReads', 'data off bins')


class TorchDevice:
    """Device buffers as torch tensors on the current CUDA device; work on torch.cuda.current_stream()."""

    def __init__(self):
        import torch
        self.torch = torch
        self.dtypes = {np.uint8: torch.uint8, np.int32: torch.int32, np.int64: torch.int64}

    def empty(self, n, dtype):
        return self.torch.empty(int(n), dtype=self.dtypes[dtype], device='cuda')

    def ptr(self, t):
        return t.data_ptr() if t is not None else 0

    def numel(self, t):
        return t.numel()

    def head(self, t, n):
        return t[:int(n)]

    def stream(self):
        return self.torch.cuda.current_stream().cuda_stream

    def upload(self, arr):
        return self.torch.from_numpy(np.ascontiguousarray(arr)).to('cuda')

    def host(self, t):
        return t.cpu().numpy()

    def upload_bytes(self, data):
        """host bytes -> a uint8 CUDA tensor, through a pinned staging tensor (the upload is then plain DMA)"""
        torch = self.torch
        src = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data).view(np.uint8)
        out = torch.empty(len(src), dtype=torch.uint8, device='cuda')
        if len(src):
            staged = torch.empty(len(src), dtype=torch.uint8, pin_memory=True)
            staged.numpy()[:] = src
            out.copy_(staged, non_blocking=True)
        return out

    def download(self, t):
        """a device tensor -> host numpy array, through a pinned tensor (one copy)"""
        staged = self.torch.empty(t.numel(), dtype=t.dtype, pin_memory=True)
        staged.copy_(t)
        return staged.numpy()

    def check(self, seq, seq_off, qual):
        torch = self.torch
        for name, t, dt in (('seq', seq, torch.uint8), ('seq_off', seq_off, torch.int64), ('qual', qual, torch.uint8)):
            if t is None:
                continue
            if not (t.is_cuda and t.dtype == dt and t.dim() == 1 and t.is_contiguous()):
                raise ValueError('%s must be a contiguous 1-D %s CUDA tensor' % (name, dt))
        if qual is not None and qual.numel() != seq.numel():
            raise ValueError('qual must hold one quality per base, at the offsets of the reads')

    def check_bytes(self, data):
        if not (data.is_cuda and data.dtype == self.torch.uint8 and data.dim() == 1 and data.is_contiguous()):
            raise ValueError('data must be a contiguous 1-D torch.uint8 CUDA tensor')

    def check_names(self, names, name_off, rna):
        torch = self.torch
        for name, t, dts in (('names', names, (torch.uint8,)), ('name_off', name_off, (torch.int64,)),
                             ('rna', rna, (torch.bool, torch.uint8))):
            if t is None:
                continue
            if not (t.is_cuda and t.dtype in dts and t.dim() == 1 and t.is_contiguous()):
                raise ValueError('%s must be a contiguous 1-D %s CUDA tensor' % (name, ' or '.join(str(d) for d in dts)))


_device = None


def device():
    """the allocator trim_reads uses (a TorchDevice unless replaced)"""
    global _device
    if _device is None:
        _device = TorchDevice()
    return _device


def initial_parts_cap(n):
    """room for output records of the first attempt: every read plus a quarter split once (chimeras are a few per cent), then
    one more call with the exact count when that is not enough"""
    return n + n // 4 + 1024


def trim_reads(seq, seq_off, matching_sets, scoring_scheme_vals, qual=None, *, end_size=150, extra_end_trim=2,
               end_threshold=75.0, min_trim_size=4, no_split=False, middle_threshold=85.0, extra_middle_trim_good_side=10,
               extra_middle_trim_bad_side=100, min_split_read_size=1000, discard_middle=False, untrimmed=False, barcodes=None):
    """What `porechop` writes for reads in GPU memory, in GPU memory.  seq: uint8 bases, seq_off: int64[n + 1] offsets, qual:
    uint8 qualities at the same offsets or None (FASTA); matching_sets and the options as for fastq.trim_fastq /
    fastq.demux_fastq.  barcodes = dict(forward_or_reverse, barcode_threshold, barcode_diff, require_two_barcodes) also calls
    the barcodes (determine_barcode) from the device's top-2 ranking.
    Returns TrimmedReads: seq, qual (None without input qualities), off (int64[n_parts + 1]), read, part (int32[n_parts]) on
    the device; start_trim / end_trim (host int32[n]), hits ({read: [(adapter position, start, end, score), ...]} as
    fastq.find_middle_hits returns them) and calls (list of bin names, or None without barcodes)."""
    D = device()
    if hasattr(D, 'check'):
        D.check(seq, seq_off, qual)
    n = D.numel(seq_off) - 1
    n_bytes = D.numel(seq)
    sets, starts, ends, adapters, left, right = _options(matching_sets, no_split, extra_middle_trim_good_side,
                                                         extra_middle_trim_bad_side)
    s_cols, e_cols, su, eu = ([], [], [], []) if barcodes is None else \
        fastq.barcode_columns(sets, barcodes.get('forward_or_reverse', 'forward'))
    pk = lambda x: W.pack_sequences(x, offset_dtype=np.int32)     # noqa: E731
    middle = pk([a[1] for a in adapters]) if adapters else None
    cap = initial_parts_cap(n)
    for attempt in range(2):
        out_seq = D.empty(max(n_bytes, 1), np.uint8)
        out_qual = D.empty(max(n_bytes, 1), np.uint8) if qual is not None else None
        out_off, out_read, out_part = D.empty(cap + 1, np.int64), D.empty(max(cap, 1), np.int32), D.empty(max(cap, 1), np.int32)
        try:
            st, et, ss, es, n_hits, h, n_parts, n_out = W.adapter_trim_split_reads_device(
                D.ptr(seq), D.ptr(seq_off), n, n_bytes, -1, pk(starts) + (s_cols,), pk(ends) + (e_cols,), middle,
                scoring_scheme_vals, end_size, extra_end_trim, end_threshold, min_trim_size, middle_threshold,
                want_top2=barcodes is not None, stream_ptr=D.stream(), d_quals_ptr=D.ptr(qual),
                mid_extra=(left, right) if adapters else None, min_split_read_size=min_split_read_size,
                discard_middle=discard_middle, untrimmed=untrimmed, d_out_seq_ptr=D.ptr(out_seq), d_out_qual_ptr=D.ptr(out_qual),
                d_out_off_ptr=D.ptr(out_off), d_out_read_ptr=D.ptr(out_read), d_out_part_ptr=D.ptr(out_part), parts_cap=cap)
        except W.EngineError as e:
            if e.code == W.ERR_SPACE and attempt == 0 and getattr(e, 'n_parts', 0) > cap:
                cap = e.n_parts                       # the exact number of records: one more call
                continue
            raise
        break
    calls = None
    if barcodes is not None:
        calls = fastq.call_barcodes_top2((su, fastq.Top2Scores(su, ss).ranked()), (eu, fastq.Top2Scores(eu, es).ranked()),
                                         barcodes.get('barcode_threshold', 75.0), barcodes.get('barcode_diff', 5.0),
                                         barcodes.get('require_two_barcodes', False))
    return TrimmedReads(D.head(out_seq, n_out), D.head(out_qual, n_out) if out_qual is not None else None,
                        D.head(out_off, n_parts + 1), D.head(out_read, n_parts), D.head(out_part, n_parts), st, et,
                        fastq._hits_dict(n_hits, h), calls)


def _options(matching_sets, no_split, extra_middle_trim_good_side, extra_middle_trim_bad_side):
    """normalised sets, start / end adapters, middle adapters and their extra trims (middle_trim_ranges: the bad side is
    before a start sequence's hit and after an end sequence's hit)"""
    sets = fastq._norm_sets(matching_sets)
    starts = [s[1] for _, s, _ in sets if s]
    ends = [e[1] for _, _, e in sets if e]
    adapters = [] if no_split else fastq._middle_adapters(sets)
    start_names, end_names = {s[0] for _, s, _ in sets if s}, {e[0] for _, _, e in sets if e}
    left = [extra_middle_trim_bad_side if nm in start_names else extra_middle_trim_good_side for nm, _ in adapters]
    right = [extra_middle_trim_bad_side if nm in end_names else extra_middle_trim_good_side for nm, _ in adapters]
    return sets, starts, ends, adapters, left, right


def demux_reads(seq, seq_off, matching_sets, scoring_scheme_vals, qual=None, *, forward_or_reverse, barcode_threshold,
                barcode_diff, require_two_barcodes, discard_unassigned, albacore_calls=None, end_size=150, extra_end_trim=2,
                end_threshold=75.0, min_trim_size=4, no_split=False, middle_threshold=85.0, extra_middle_trim_good_side=10,
                extra_middle_trim_bad_side=100, min_split_read_size=1000, discard_middle=False, untrimmed=False):
    """What `porechop -b DIR` writes for reads in GPU memory, in GPU memory and grouped by bin (one
    adapterDemuxReadsDevice call).  Arguments as trim_reads, plus the barcode options of fastq.demux_fastq; albacore_calls:
    one bin name (or None) per read, or None.
    Returns DemuxedReads: seq, qual, off, read, part on the device as in trim_reads, with the records grouped by bin (bins in
    the order of the barcode names, 'none' last; read order inside a bin); bins = {name: (first record, end record)} for the
    bins that have records; calls (one bin name per read, demux_fastq's info['calls']); start_trim / end_trim / hits as
    trim_reads returns them."""
    D = device()
    if hasattr(D, 'check'):
        D.check(seq, seq_off, qual)
    n = D.numel(seq_off) - 1
    n_bytes = D.numel(seq)
    sets, starts, ends, adapters, left, right = _options(matching_sets, no_split, extra_middle_trim_good_side,
                                                         extra_middle_trim_bad_side)
    s_cols, e_cols, su, eu = fastq.barcode_columns(sets, forward_or_reverse)
    names = list(dict.fromkeys(su + eu))
    idx = {nm: i for i, nm in enumerate(names)}
    n_bins = len(names)
    alb = None
    if albacore_calls is not None:
        if len(albacore_calls) != n:
            raise ValueError('albacore_calls needs one entry per read')
        alb = D.upload(np.array([-1 if a is None else idx.get(a, n_bins + 1) for a in albacore_calls], dtype=np.int32))
    pk = lambda x: W.pack_sequences(x, offset_dtype=np.int32)     # noqa: E731
    middle = pk([a[1] for a in adapters]) if adapters else None
    cap = initial_parts_cap(n)
    for attempt in range(2):
        out_seq = D.empty(max(n_bytes, 1), np.uint8)
        out_qual = D.empty(max(n_bytes, 1), np.uint8) if qual is not None else None
        out_off, out_read, out_part = D.empty(cap + 1, np.int64), D.empty(max(cap, 1), np.int32), D.empty(max(cap, 1), np.int32)
        try:
            st, et, n_hits, h, n_parts, n_out, read_bin, bin_parts = W.adapter_demux_reads_device(
                D.ptr(seq), D.ptr(seq_off), n, n_bytes, -1, pk(starts) + (s_cols,), pk(ends) + (e_cols,), middle,
                scoring_scheme_vals, end_size, extra_end_trim, end_threshold, min_trim_size, middle_threshold,
                stream_ptr=D.stream(), start_bin=[idx[nm] for nm in su], end_bin=[idx[nm] for nm in eu], n_bins=n_bins,
                barcode_threshold=barcode_threshold, barcode_diff=barcode_diff, require_two_barcodes=require_two_barcodes,
                discard_unassigned=discard_unassigned, d_albacore_ptr=D.ptr(alb), d_quals_ptr=D.ptr(qual),
                mid_extra=(left, right) if adapters else None, min_split_read_size=min_split_read_size,
                discard_middle=discard_middle, untrimmed=untrimmed, d_out_seq_ptr=D.ptr(out_seq), d_out_qual_ptr=D.ptr(out_qual),
                d_out_off_ptr=D.ptr(out_off), d_out_read_ptr=D.ptr(out_read), d_out_part_ptr=D.ptr(out_part), parts_cap=cap)
        except W.EngineError as e:
            if e.code == W.ERR_SPACE and attempt == 0 and getattr(e, 'n_parts', 0) > cap:
                cap = e.n_parts                       # the exact number of records: one more call
                continue
            raise
        break
    bin_names = names + ['none']
    bins = {bin_names[b]: (int(bin_parts[b]), int(bin_parts[b + 1])) for b in range(n_bins + 1) if bin_parts[b + 1] > bin_parts[b]}
    return DemuxedReads(D.head(out_seq, n_out), D.head(out_qual, n_out) if out_qual is not None else None,
                        D.head(out_off, n_parts + 1), D.head(out_read, n_parts), D.head(out_part, n_parts), bins,
                        [bin_names[b] for b in read_bin.tolist()], st, et, fastq._hits_dict(n_hits, h))


def initial_out_cap(n_rec, n_bases, longest_name, fmt):
    """room for the output bytes of the first attempt: an upper bound -- the bases (and qualities), then per record the longest
    name, an 11-byte part tag ('_' and up to 10 digits) and the fixed bytes (FASTQ '@', '\\n', '\\n+\\n', '\\n'; FASTA '>', '\\n'
    and at most one more line end than n_bases / 70)"""
    if fmt == 'fastq':
        return 2 * n_bases + n_rec * (longest_name + 11 + 6)
    return n_bases + n_bases // 70 + n_rec * (longest_name + 11 + 3)


def emit_reads(out, names, name_off, rna=None, fmt='fastq'):
    """The bytes Porechop writes for the records of trim_reads / demux_reads (a TrimmedReads or DemuxedReads), formatted on the
    device (pb200EmitReadsDevice): the bytes fastq.emit_parts writes for the same records.  names (uint8) / name_off
    (int64[n_reads + 1]): the source reads' names; rna: bool or uint8 per read (RNA reads are written with U), or None.
    fmt: 'fastq' or 'fasta'.
    Returns EmittedReads: data (uint8, exactly the output's length) and off (int64[n_records + 1], record byte offsets) on the
    device; bins = {name: (first byte, end byte)} of every bin of a DemuxedReads -- each bin's file is one slice of data --
    or None for a TrimmedReads."""
    if fmt not in ('fastq', 'fasta'):
        raise ValueError("fmt must be 'fastq' or 'fasta'")
    if fmt == 'fastq' and out.qual is None:
        raise ValueError('FASTQ output needs the qualities')
    D = device()
    if hasattr(D, 'check_names'):
        D.check_names(names, name_off, rna)
    n_rec, n_reads = D.numel(out.read), D.numel(name_off) - 1
    if n_reads < 0 or (rna is not None and D.numel(rna) != n_reads):
        raise ValueError('name_off needs n_reads + 1 offsets and rna one flag per read')
    name_len = np.diff(D.host(name_off))
    cap = initial_out_cap(n_rec, D.numel(out.seq), int(name_len.max()) if len(name_len) else 0, fmt)
    off = D.empty(n_rec + 1, np.int64)
    for attempt in range(2):
        data = D.empty(max(cap, 1), np.uint8)
        try:
            n_out = W.pb200_emit_reads_device(
                n_rec, d_seq_ptr=D.ptr(out.seq), d_qual_ptr=D.ptr(out.qual) if fmt == 'fastq' else 0, seq_bytes=D.numel(out.seq),
                d_off_ptr=D.ptr(out.off), d_read_ptr=D.ptr(out.read), d_part_ptr=D.ptr(out.part), d_names_ptr=D.ptr(names),
                d_name_off_ptr=D.ptr(name_off), n_reads=n_reads, name_bytes=D.numel(names), d_rna_ptr=D.ptr(rna), fmt=fmt,
                d_out_ptr=D.ptr(data), out_cap=cap, d_out_off_ptr=D.ptr(off), stream_ptr=D.stream())
        except W.EngineError as e:
            if e.code == W.ERR_SPACE and attempt == 0 and getattr(e, 'n_out_bytes', 0) > cap:
                cap = e.n_out_bytes                   # the exact number of bytes: one more call
                continue
            raise
        break
    bins = None
    if isinstance(out, DemuxedReads):
        o = D.host(off)
        bins = {name: (int(o[r0]), int(o[r1])) for name, (r0, r1) in out.bins.items()}
    return EmittedReads(D.head(data, n_out), off, bins)


# ---- bytes in: FASTQ / FASTA parsed on the device, and whole chunks from input bytes to output bytes ------------------------
ParsedReads = collections.namedtuple('ParsedReads', 'names name_off seq seq_off qual rna kind')

_PARSE_MESSAGES = {W.PARSE_LINES: 'FASTQ chunk is not a whole number of 4-line records',
                   W.PARSE_HEADER: 'FASTQ record does not start with @',
                   W.PARSE_FASTA_START: 'FASTA does not start with a > line',
                   W.PARSE_FASTA_NAME: 'FASTA record with an empty name'}


class QualityTooLong(ValueError):
    """a FASTQ quality line is longer than its bases: the device layout keeps one quality per base at the bases' offsets, so
    the chunk is parsed on the host instead (fastq.parse_fastq keeps such qualities as they are).  .index: the read."""

    def __init__(self, index):
        super().__init__('read %d has a quality line longer than its bases' % index)
        self.index = index


def initial_parse_caps(n_bytes, kind):
    """(reads, name bytes, bases) of the first attempt of parse_reads for n_bytes of input: the bases fit in any case, names and
    reads fit unless records average under 32 bytes; otherwise one more call with the exact counts"""
    return n_bytes // 32 + 64, n_bytes // 4 + 4096, n_bytes


def _kind_of(D, data, n):
    """FASTQ or FASTA by the first byte, like fastq.parse_reads (get_sequence_file_type, misc.py:84-106)"""
    head = bytes(D.host(D.head(data, 1))) if n else b''
    if head == b'>':
        return 'fasta'
    if head in (b'@', b''):
        return 'fastq'
    raise ValueError('File is neither FASTA or FASTQ')


def parse_reads(data, kind=None, qual=True):
    """FASTQ / FASTA bytes in GPU memory -> the reads in GPU memory (pb200ParseReadsDevice): the fields fastq.parse_fastq /
    fastq.parse_fasta return, field for field.  data: contiguous 1-D uint8 CUDA tensor of whole records; kind: 'fastq',
    'fasta' or None (from the first byte, as fastq.parse_reads); qual=False writes no qualities (FASTA output).
    Returns ParsedReads(names, name_off, seq, seq_off, qual, rna, kind) on the device -- the arguments trim_reads, demux_reads
    and emit_reads take; qual is None when not asked for.  Malformed input raises the host parser's ValueError; a FASTQ quality
    line longer than its bases raises QualityTooLong (with qual=True)."""
    D = device()
    if hasattr(D, 'check_bytes'):
        D.check_bytes(data)
    n = D.numel(data)
    if kind is None:
        kind = _kind_of(D, data, n)
    if kind not in ('fastq', 'fasta'):
        raise ValueError("kind must be 'fastq', 'fasta' or None")
    reads_cap, names_cap, seq_cap = initial_parse_caps(n, kind)
    for attempt in range(2):
        names, seq = D.empty(max(names_cap, 1), np.uint8), D.empty(max(seq_cap, 1), np.uint8)
        q = D.empty(max(seq_cap, 1), np.uint8) if qual else None
        name_off, seq_off = D.empty(reads_cap + 1, np.int64), D.empty(reads_cap + 1, np.int64)
        rna = D.empty(max(reads_cap, 1), np.uint8)
        try:
            n_reads, n_names, n_seq = W.pb200_parse_reads_device(
                D.ptr(data), n, kind, d_names_ptr=D.ptr(names), names_cap=names_cap, d_name_off_ptr=D.ptr(name_off),
                d_seq_ptr=D.ptr(seq), seq_cap=seq_cap, d_seq_off_ptr=D.ptr(seq_off), d_qual_ptr=D.ptr(q), d_rna_ptr=D.ptr(rna),
                reads_cap=reads_cap, stream_ptr=D.stream())
        except W.EngineError as e:
            if e.code == W.ERR_SPACE and attempt == 0:
                reads_cap, names_cap, seq_cap = e.n_reads, e.n_name_bytes, e.n_seq_bytes    # the exact counts: one more call
                continue
            reason = getattr(e, 'reason', 0)
            if reason in _PARSE_MESSAGES:
                raise ValueError(_PARSE_MESSAGES[reason]) from None
            if reason == W.PARSE_LONG_QUAL:
                raise QualityTooLong(e.index) from None
            raise
        break
    return ParsedReads(D.head(names, n_names), D.head(name_off, n_reads + 1), D.head(seq, n_seq), D.head(seq_off, n_reads + 1),
                       D.head(q, n_seq) if qual else None, D.head(rna, n_reads), kind)


def _upload(D, data):
    up = getattr(D, 'upload_bytes', None)
    if up is not None:
        return up(data)
    return D.upload(np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data)


def _host_batch(data, kind):
    if kind is None:
        return fastq.parse_reads(data)[0]
    return fastq.parse_fasta(data) if kind == 'fasta' else fastq.parse_fastq(data)


def _device_chunk(data, kind, matching_sets, fmt, end_threshold, run):
    """upload -> parse_reads -> run(parsed) -> emit_reads; None when the host path must take this chunk (a quality line longer
    than its bases, no reads, nothing to align, or inputs the device call does not take: PB200_ERR_ARG)"""
    if fmt not in ('fastq', 'fasta'):
        raise ValueError("fmt must be 'fastq' or 'fasta'")
    sets = fastq._norm_sets(matching_sets)
    if end_threshold < 0 or not any(s or e for _, s, e in sets):
        return None
    D = device()
    d_in = _upload(D, data)
    try:
        p = parse_reads(d_in, kind, qual=fmt == 'fastq')
    except QualityTooLong:
        return None
    n = D.numel(p.rna)
    if n == 0:
        return None
    try:
        out = run(p, n)
    except W.EngineError as e:
        if e.code != W.ERR_ARG:
            raise
        return None
    em = emit_reads(out, p.names, p.name_off, p.rna, fmt)
    return out, em, getattr(D, 'download', D.host)(em.data), n


def trim_fastq(data, matching_sets, scoring_scheme_vals, end_size=150, extra_end_trim=2, end_threshold=75.0, min_trim_size=4,
               no_split=False, middle_threshold=85.0, extra_middle_trim_good_side=10, extra_middle_trim_bad_side=100,
               min_split_read_size=1000, discard_middle=False, fmt='fastq', as_array=False, kind=None):
    """fastq.trim_fastq on the device from input bytes to output bytes: host bytes of whole FASTQ / FASTA records (kind: 'fastq',
    'fasta' or None = from the first byte) go up once, parse_reads -> trim_reads -> emit_reads run in GPU memory, and the output
    bytes come home in one copy.  Returns (output bytes, or a uint8 array with as_array; info with start_trim, end_trim and
    n_reads) -- the bytes fastq.trim_fastq writes for the parsed reads.  A chunk the device path does not take (a quality line
    longer than its bases, inputs adapterTrimSplitReadsDevice refuses) runs through fastq.trim_fastq instead, with the same
    result.  Malformed input raises the host parser's ValueError."""
    opts = dict(end_size=end_size, extra_end_trim=extra_end_trim, end_threshold=end_threshold, min_trim_size=min_trim_size,
                no_split=no_split, middle_threshold=middle_threshold, extra_middle_trim_good_side=extra_middle_trim_good_side,
                extra_middle_trim_bad_side=extra_middle_trim_bad_side, min_split_read_size=min_split_read_size,
                discard_middle=discard_middle)
    got = _device_chunk(data, kind, matching_sets, fmt, end_threshold,
                        lambda p, n: trim_reads(p.seq, p.seq_off, matching_sets, scoring_scheme_vals, p.qual, **opts))
    if got is None:
        return fastq.trim_fastq(_host_batch(data, kind), matching_sets, scoring_scheme_vals, fmt=fmt, as_array=as_array, **opts)
    out, _, host, n = got
    info = {'start_trim': np.asarray(out.start_trim, dtype=np.int64), 'end_trim': np.asarray(out.end_trim, dtype=np.int64),
            'hits': out.hits, 'n_reads': n}
    return (host if as_array else host.tobytes()), info


def demux_fastq(data, matching_sets, scoring_scheme_vals, forward_or_reverse='forward', end_size=150, extra_end_trim=2,
                end_threshold=75.0, min_trim_size=4, no_split=False, middle_threshold=85.0, extra_middle_trim_good_side=10,
                extra_middle_trim_bad_side=100, min_split_read_size=1000, discard_middle=False, barcode_threshold=75.0,
                barcode_diff=5.0, require_two_barcodes=False, discard_unassigned=False, untrimmed=False, fmt='fastq',
                albacore_calls=None, as_array=False, kind=None):
    """fastq.demux_fastq on the device from input bytes to output bytes, as trim_fastq: parse_reads -> demux_reads -> emit_reads,
    and every bin's bytes are one slice of the single copy home.  albacore_calls: one bin name (or None) per read, one name for
    every read, or None.  Returns ({bin name: bytes (or uint8 arrays with as_array)}, info with calls, start_trim, end_trim and
    n_reads); chunks the device path does not take run through fastq.demux_fastq, with the same result."""
    opts = dict(end_size=end_size, extra_end_trim=extra_end_trim, end_threshold=end_threshold, min_trim_size=min_trim_size,
                no_split=no_split, middle_threshold=middle_threshold, extra_middle_trim_good_side=extra_middle_trim_good_side,
                extra_middle_trim_bad_side=extra_middle_trim_bad_side, min_split_read_size=min_split_read_size,
                discard_middle=discard_middle, untrimmed=untrimmed)
    bc = dict(forward_or_reverse=forward_or_reverse, barcode_threshold=barcode_threshold, barcode_diff=barcode_diff,
              require_two_barcodes=require_two_barcodes, discard_unassigned=discard_unassigned)

    def calls_for(n):
        return [albacore_calls] * n if isinstance(albacore_calls, str) else albacore_calls
    got = _device_chunk(data, kind, matching_sets, fmt, end_threshold,
                        lambda p, n: demux_reads(p.seq, p.seq_off, matching_sets, scoring_scheme_vals, p.qual,
                                                 albacore_calls=calls_for(n), **bc, **opts))
    if got is None:
        batch = _host_batch(data, kind)
        return fastq.demux_fastq(batch, matching_sets, scoring_scheme_vals, fmt=fmt, albacore_calls=calls_for(len(batch)),
                                 as_array=as_array, **bc, **opts)
    out, em, host, n = got
    bins = {name: host[b0:b1] if as_array else host[b0:b1].tobytes() for name, (b0, b1) in em.bins.items()}
    info = {'start_trim': np.asarray(out.start_trim, dtype=np.int64), 'end_trim': np.asarray(out.end_trim, dtype=np.int64),
            'hits': out.hits, 'calls': out.calls, 'n_reads': n}
    return bins, info
