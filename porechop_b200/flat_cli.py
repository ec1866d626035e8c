"""
`python -m porechop_b200.flat_cli <porechop arguments>`: Porechop's run on flat buffers (no per-read Python objects).

The argument parser, the adapter table and every policy decision are the user's Porechop checkout's own code, called
as is (`porechop.porechop.get_arguments`, `ADAPTERS`, `fix_up_1d2_sets`, `choose_barcoding_kit`,
`add_full_barcode_adapter_sets`; porechop.py:33-79).  What is replaced is the data path between them
(porechop_b200/fastq.py): FASTQ bytes -> flat buffers -> batched alignments on the engine -> trim / split / barcode
decisions on arrays -> output bytes.  Output files are byte-identical to the reference CLI's
(tests/test_flat_cli.py); the progress / verbose report is not reproduced -- use `python -m porechop_b200`
(porechop_b200/patch.py) when that is wanted.

The input is streamed in whole-record chunks (PB200_FLAT_CHUNK_BYTES, default 256 MB; the first chunk holds the check
reads of Phase A), so memory is bounded by the chunk size, not the file size.

Opt-in device paths (environment, off by default; output bytes are the same): PB200_DEVICE_DECISIONS=1 runs the end-trim
decisions on the device (adapterEndDecisions), PB200_DEVICE_MIDDLE=1 runs the whole middle-adapter scan there, masking
rounds included (adapterMiddleScan; inputs it does not take -- e.g. adapters with other bases than A/C/G/T/U -- use the
host rounds), PB200_CHECK_ALL_READS=1 runs Phase A over every read, and PB200_DEVICE_SEARCH=1 reduces Phase A's records to
one best score per adapter sequence on the device (adapterSetSearch) -- what makes checking every read cheap.  With
PB200_DEVICE_DECISIONS=1 and PB200_DEVICE_MIDDLE=1 both set, each chunk's Phase B and Phase C are one engine call
(adapterTrimReads): the reads are uploaded once and the windows, trims and trimmed reads are made on the device.
PB200_DEVICE_READS=1 takes each chunk from input bytes to output bytes on the device (device_reads.trim_fastq /
demux_fastq): the raw bytes go up, are parsed there (pb200ParseReadsDevice), trimmed, split or demultiplexed and formatted
there, and the output bytes come home in one copy; the background thread only reads (and gunzips) the input.  Chunks with
nothing to align (no adapter set matched) and Phase A keep the host parse.  With PB200_DEVICE_READS=1, PB200_DEVICE_GZIP=1
also compresses a .gz output on the device (device_reads.gzip_bytes: 64 KiB gzip members, a ratio between zlib's levels 1
and 6 is not promised) before the one copy home; chunks with nothing to align are still compressed by the host.  It is a
trade of compression ratio against time, like PB200_GZIP_LEVEL, so it stays the user's choice.

Multi-GPU: launched with torchrun (one process per GPU) chunk c is handled by rank c % world on its own device; ranks
write self-contained pieces and rank 0 stitches them in chunk order after a barrier -- no data-path collective
(SURVEY 8e).

Input: one FASTQ or FASTA file (plain or .gz), or an Albacore output directory of FASTQ files (porechop.py:224-273).
"""
import gzip
import os
import sys

from . import fastq, hostio


def _record_chunks(path, chunk_bytes, first_reads):
    """Whole-record pieces of a FASTQ / FASTA file (plain or .gz): the first piece holds at least `first_reads` reads
    (Phase A's check reads, porechop.py:237), the others about chunk_bytes each, so a run's memory is bounded by the
    chunk size.  Yields (kind, bytes) with kind 'fastq' | 'fasta' from the file's first character (misc.py:84-106)."""
    with open(path, 'rb') as f:
        magic = f.read(2)
    opener = gzip.open if magic == b'\x1f\x8b' else open
    with opener(path, 'rb') as f:
        pending, first, kind = b'', True, None
        while True:
            block = f.read(chunk_bytes)
            data = pending + block
            if kind is None:
                kind = {b'>': 'fasta', b'@': 'fastq', b'': 'fastq'}.get(data[:1])
                if kind is None:
                    sys.exit('porechop_b200.flat_cli: ' + path + ' is neither FASTA nor FASTQ')
            if not block:
                if data.strip() or first:
                    yield kind, data
                return
            if kind == 'fasta':                             # records start at a '>' that begins a line
                cut = data.rfind(b'\n>') + 1
                n_rec = data.count(b'\n>', 0, cut) + 1 if cut else 0
            else:
                cut = data.rfind(b'\n') + 1                 # drop the unterminated last line
                n_nl = data.count(b'\n', 0, cut)
                for _ in range(n_nl % 4):                   # back to a multiple of four lines
                    cut = data.rfind(b'\n', 0, cut - 1) + 1
                n_rec = n_nl // 4
            if cut == 0 or (first and n_rec < first_reads):
                pending = data                              # keep reading (Phase A wants its check reads in one piece)
                continue
            yield kind, data[:cut]
            pending, first = data[cut:], False


def _prefetch(it, depth=2):
    """Run an iterator in a background thread, `depth` items ahead: reading, gunzipping and parsing the next chunk
    (zlib, libhostio and the engine all release the GIL) overlaps the alignment and the writing of the current one."""
    import queue
    import threading
    q, end = queue.Queue(maxsize=depth), object()

    def work():
        try:
            for item in it:
                q.put(item)
            q.put(end)
        except BaseException as e:          # re-raised in the consumer (sys.exit from the reader included)
            q.put(e)
    threading.Thread(target=work, daemon=True).start()
    while True:
        item = q.get()
        if item is end:
            return
        if isinstance(item, BaseException):
            raise item
        yield item


class _Sink:
    """one output stream (file, gz file or stdout), opened on first write like the reference's bin files.
    A .gz stream is written as independent gzip members (block-parallel deflate in libhostio.so, or the gzip module):
    the same bytes after decompression as the reference's `gzip -c` / `pigz`.
    With world > 1 every rank writes its pieces to `<path>.rank<r>` and remembers (chunk index, offset, length);
    rank 0 stitches the pieces of all ranks together in chunk order afterwards (`_merge_rank_files`)."""

    def __init__(self, path, gz, rank=0, world=1):
        self.final, self.gz, self.f, self.ranked = path, gz, None, world > 1
        self.path = path if not self.ranked else '%s.rank%d' % (path, rank)
        self.index = []                                    # ranked mode: [chunk, offset, length]

    def write(self, payload, chunk=0, packed=False):
        """packed: payload is already gzip members (compressed on the device) and is written as it is"""
        if not len(payload):
            return
        if self.f is None:
            self.f = sys.stdout.buffer if self.final is None else open(self.path, 'wb')
        if self.gz and not packed:
            level = int(os.environ.get('PB200_GZIP_LEVEL', 6))
            packed = hostio.gzip_members(payload, level)
            payload = packed if packed is not None else gzip.compress(bytes(payload), level)
        start = self.f.tell() if self.ranked else 0
        self.f.write(payload)
        if self.ranked:
            self.index.append([chunk, start, self.f.tell() - start])

    def close(self):
        if self.f is not None and self.final is not None:
            self.f.close()


def _merge_rank_files(final_paths, world):
    """rank 0, after the barrier: final file = the pieces of all ranks in chunk order (a multi-member .gz is a valid
    .gz of the concatenation); the per-rank files are removed."""
    import json
    for final in final_paths:
        pieces = []
        for r in range(world):
            idx = '%s.rank%d.idx' % (final, r)
            if os.path.exists(idx):
                pieces += [(c, r, off, ln) for c, off, ln in json.load(open(idx))]
                os.remove(idx)
        if not pieces:
            continue
        files = {r: open('%s.rank%d' % (final, r), 'rb') for r in {p[1] for p in pieces}}
        with open(final, 'wb') as out:
            for c, r, off, ln in sorted(pieces):
                files[r].seek(off)
                out.write(files[r].read(ln))
        for r, f in files.items():
            f.close()
            os.remove('%s.rank%d' % (final, r))


def _out_format(args, read_type='fastq'):
    # the format rules of output_reads (porechop.py:624-650)
    fmt = args.format
    if fmt == 'auto':
        if args.output is None:
            fmt = read_type
            if args.barcode_dir is not None and args.input.lower().endswith('.gz'):
                fmt += '.gz'
        else:
            low = args.output.lower()
            fmt = next((f for f in ('fasta.gz', 'fastq.gz', 'fasta', 'fastq') if '.' + f in low), read_type)
    gz = fmt.endswith('.gz') and (args.barcode_dir is not None or args.output is not None)
    return (fmt[:-3] if fmt.endswith('.gz') else fmt), gz


def main():
    try:
        from porechop import porechop as P
    except ImportError:
        sys.exit('porechop_b200.flat_cli: no `porechop` package on sys.path (point PYTHONPATH at a Porechop checkout)')
    args = P.get_arguments()
    scoring = args.scoring_scheme_vals
    chunk_bytes = int(os.environ.get('PB200_FLAT_CHUNK_BYTES', 256 << 20))
    # one process per GPU (torchrun): chunk c belongs to rank c % world; nothing but a final barrier is exchanged
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    device_reads = None
    if os.environ.get('PB200_DEVICE_READS', '0') == '1':
        from . import device_reads
    device_gzip = device_reads is not None and os.environ.get('PB200_DEVICE_GZIP', '0') == '1'
    if world > 1:
        import torch.distributed as dist
        from . import cpp_function_wrappers as W
        if args.output is None and args.barcode_dir is None:
            sys.exit('porechop_b200.flat_cli: multi-process runs need -o or -b (stdout cannot be stitched)')
        n_dev = W.device_count()
        if n_dev > 0:
            W.set_device(int(os.environ.get('LOCAL_RANK', rank)) % n_dev)
            if device_reads is not None:        # device_reads allocates on torch's current device: the engine's
                import torch
                torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', rank)) % n_dev)
        dist.init_process_group('gloo')                   # host-side barrier only; the data path has no collective
        local_world = int(os.environ.get('LOCAL_WORLD_SIZE', world))
        hostio.set_threads(max(1, hostio.usable_cpus() // max(local_world, 1)))    # torchrun exports OMP_NUM_THREADS=1
    if os.path.isdir(args.input):
        # an Albacore output directory (porechop.py:241-266): every *.fastq[.gz] below it in sorted order, the check
        # reads spread over the files, and Albacore's own bin (from the path) must agree with the barcode call
        inputs = sorted(os.path.join(d, f) for d, _, names in os.walk(args.input) for f in names
                        if f.lower().endswith('.fastq') or f.lower().endswith('.fastq.gz'))
        if not inputs:
            sys.exit('Error: could not find fastq files in ' + args.input)
        check_per_file = int(round(args.check_reads / len(inputs)))
        albacore = [P.get_albacore_barcode_from_path(f) for f in inputs]
    elif os.path.isfile(args.input):
        inputs, check_per_file, albacore = [args.input], args.check_reads, [None]
    else:
        sys.exit('Error: could not find ' + args.input)
    parsers = {'fasta': fastq.parse_fasta, 'fastq': fastq.parse_fastq}

    # Phase A on flat buffers; the scores land on Porechop's own Adapter objects so that its policy code runs unchanged
    search = [a for a in P.ADAPTERS if '(full sequence)' not in a.name]                     # porechop.py:296
    as_tuple = lambda a: (a.name, tuple(a.start_sequence) or None, tuple(a.end_sequence) or None)   # noqa: E731
    read_type = 'fastq'
    # PB200_CHECK_ALL_READS=1 (opt-in, SURVEY 8(f) row 4; the reference's README suggests a larger --check_reads when adapters
    # are rare): Phase A looks at EVERY read instead of the first --check_reads -- one extra streaming pass over the input
    # in the same bounded chunks; a set's best score is a maximum, so chunks (and ranks) combine exactly.
    check_all = os.environ.get('PB200_CHECK_ALL_READS', '0') == '1'
    sets_a = [as_tuple(a) for a in search]

    def note(best_s, best_e):
        for a, s, e in zip(search, best_s, best_e):
            a.best_start_score, a.best_end_score = max(a.best_start_score, float(s)), max(a.best_end_score, float(e))
    chunk_no = 0
    for path in inputs:
        if check_all:
            for kind, data in _record_chunks(path, chunk_bytes, 0):
                if len(inputs) == 1:
                    read_type = kind
                if chunk_no % world == rank:
                    batch = parsers[kind](data)
                    note(*fastq.search_adapter_sets(batch, sets_a, scoring, len(batch), args.end_size))
                chunk_no += 1
            continue
        kind, first = next(_record_chunks(path, chunk_bytes, check_per_file))
        if len(inputs) == 1:
            read_type = kind
        if check_per_file <= 0:
            continue
        note(*fastq.search_adapter_sets(parsers[kind](first), sets_a, scoring, check_per_file, args.end_size))
    if check_all and world > 1:          # every rank saw its own chunks: the per-set maxima are combined (host-side, gloo)
        mine = [(a.best_start_score, a.best_end_score) for a in search]
        every = [None] * world
        dist.all_gather_object(every, mine)
        for k, a in enumerate(search):
            a.best_start_score = max(r[k][0] for r in every)
            a.best_end_score = max(r[k][1] for r in every)
    matching = [a for a in search if a.best_start_or_end_score() >= args.adapter_threshold]  # porechop.py:327
    matching = P.fix_up_1d2_sets(matching)
    null = open(os.devnull, 'w')
    direction = P.choose_barcoding_kit(matching, 0, null) if args.barcode_dir else None
    matching = P.add_full_barcode_adapter_sets(matching)
    sets = [as_tuple(a) for a in matching]

    fmt, gz = _out_format(args, read_type)
    common = dict(end_size=args.end_size, extra_end_trim=args.extra_end_trim, end_threshold=args.end_threshold,
                  min_trim_size=args.min_trim_size, no_split=args.no_split, middle_threshold=args.middle_threshold,
                  extra_middle_trim_good_side=args.extra_middle_trim_good_side,
                  extra_middle_trim_bad_side=args.extra_middle_trim_bad_side,
                  min_split_read_size=args.min_split_read_size, discard_middle=args.discard_middle, fmt=fmt, as_array=True)
    sinks = {}

    def sink(name):
        if name not in sinks:
            path = args.output if name is None else os.path.join(args.barcode_dir, name + '.' + fmt + ('.gz' if gz else ''))
            sinks[name] = _Sink(path, gz, rank, world)
        return sinks[name]
    if args.barcode_dir is not None:
        os.makedirs(args.barcode_dir, exist_ok=True)

    def process(batch, albacore_call, chunk):
        # batch: a FastqBatch, or with PB200_DEVICE_READS=1 (kind, raw bytes) -- parsed on the host only when nothing is aligned
        on_device = device_reads is not None and sets
        packed = bool(on_device and gz and device_gzip)      # the device path's bytes come home compressed
        if device_reads is not None and not sets:
            batch = parsers[batch[0]](batch[1])
        if args.barcode_dir is None:
            if on_device:
                out, _ = device_reads.trim_fastq(batch[1], sets, scoring, kind=batch[0], gz=packed, **common)
            elif sets:
                out, _ = fastq.trim_fastq(batch, sets, scoring, **common)
            else:                   # "No adapters found - output reads are unchanged from input reads"
                out = fastq.emit(batch, fmt=fmt, as_array=True)
            sink(None).write(out, chunk, packed)
            return
        if sets:
            bc = dict(barcode_threshold=args.barcode_threshold, barcode_diff=args.barcode_diff,
                      require_two_barcodes=args.require_two_barcodes, discard_unassigned=args.discard_unassigned,
                      untrimmed=args.untrimmed)
            if on_device:
                bins, _ = device_reads.demux_fastq(batch[1], sets, scoring, direction, albacore_calls=albacore_call,
                                                   kind=batch[0], gz=packed, **bc, **common)
            else:
                calls = None if albacore_call is None else [albacore_call] * len(batch)
                bins, _ = fastq.demux_fastq(batch, sets, scoring, direction, albacore_calls=calls, **bc, **common)
        else:
            out = fastq.emit(batch, fmt=fmt, untrimmed=args.untrimmed, as_array=True)
            bins = {} if args.discard_unassigned else {'none': out}
        for name, payload in bins.items():
            sink(name).write(payload, chunk, packed)

    def batches():
        chunk = 0
        for path, albacore_call in zip(inputs, albacore):
            for kind, data in _record_chunks(path, chunk_bytes, 0):
                if chunk % world == rank:
                    yield ((kind, data) if device_reads is not None else parsers[kind](data)), albacore_call, chunk
                chunk += 1
    for batch, albacore_call, chunk in _prefetch(batches()):
        process(batch, albacore_call, chunk)
    def touch_output():                                   # an empty result is still a file (porechop.py:713-727)
        with open(args.output, 'wb') as f:
            f.write(gzip.compress(b'') if gz else b'')
    if world == 1:
        for s_ in sinks.values():
            s_.close()
        if args.barcode_dir is None and args.output is not None and (None not in sinks or sinks[None].f is None):
            touch_output()
        return 0
    import json
    for s_ in sinks.values():
        s_.close()
        if s_.index:
            json.dump(s_.index, open(s_.path + '.idx', 'w'))
    finals = [None] * world                               # which output files exist anywhere (bins differ per rank)
    dist.all_gather_object(finals, [s_.final for s_ in sinks.values()])
    dist.barrier()
    if rank == 0:
        names = sorted({f for fs in finals for f in fs})
        _merge_rank_files(names, world)
        if args.barcode_dir is None and not os.path.exists(args.output):
            touch_output()
    dist.barrier()
    dist.destroy_process_group()
    return 0


if __name__ == '__main__':
    sys.exit(main())
