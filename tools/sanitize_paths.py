#!/usr/bin/env python3
"""Small runs of every engine path (default + opt-in) for compute-sanitizer on the GPU box:

    compute-sanitizer --tool memcheck  python tools/sanitize_paths.py
    compute-sanitizer --tool racecheck python tools/sanitize_paths.py      (shared-memory hazards: staging rings, profiles)

Inputs are tiny (the tools slow kernels down by 10-100x); results are compared with the oracle so a run also fails on
wrong records.  The host simulation (tests/sim) already runs the same paths under AddressSanitizer and with shuffled lane
order; this is the hardware-side counterpart."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import numpy as np                                  # noqa: E402
from helpers import oracle_batch                    # noqa: E402
from porechop_b200 import cpp_function_wrappers as W, workloads as wl    # noqa: E402

DEFAULTS = {'h2d_pack': 0, 'tight_window': 1, 'profile': 1, 'direct_max': 160, 'chunk_tasks': 131072,
            'hbuf': 'auto'}
yt, yb = wl.nsk007()
_, sw, ew = wl.synth_end_windows(600, yt, yb, seed=1)
sbuf, soff = wl.windows_to_batch(sw)
a1, o1 = wl.pack_adapters([yt])
a2, o2 = wl.pack_adapters([yt, yb])
lbuf, loff = wl.synth_reads(6, yt, yb, seed=2, chimera_p=0.5, max_len=4000)
starts, ends = wl.demux_adapters()
bad = 0


def run(label, opts, fn):
    global bad
    try:
        for k, v in opts.items():
            W.set_option(k, v)
        got, exp = fn()
    finally:
        for k in opts:
            W.set_option(k, DEFAULTS[k])
    ok = np.array_equal(got, exp)
    bad += 0 if ok else 1
    print('%-10s %-70s %s' % (label, opts, 'ok' if ok else 'DIFFERENT'), flush=True)


def cross(buf, off, ab, ao):
    return lambda: (W.adapter_alignment_batch(buf, off, ab, ao, wl.DEFAULT_SCORING), oracle_batch(buf, off, ab, ao, wl.DEFAULT_SCORING))


for opts in ({}, {'direct_max': 100}, {'direct_max': 100, 'tight_window': 0}, {'h2d_pack': 1, 'chunk_tasks': 200},
             {'hbuf': 'global'}):
    run('windows', opts, cross(sbuf, soff, a1, o1))
    run('windows2', opts, cross(sbuf, soff, a2, o2))
for opts in ({}, {'profile': 0, 'tight_window': 0}, {'profile': 0}, {'direct_max': 100000, 'hbuf': 'global'}):
    run('long', opts, cross(lbuf, loff, a2, o2))
a3, o3 = wl.pack_adapters(starts)
run('demux', {}, cross(sbuf[:150 * 12], soff[:13], a3, o3))
run('demux', {'direct_max': 100}, cross(sbuf[:150 * 12], soff[:13], a3, o3))
run('demux', {'hbuf': 'global'}, cross(sbuf[:150 * 12], soff[:13], a3, o3))
outs = W.adapter_end_decisions([(sbuf, soff, a2, o2, True, [0, 1])], wl.DEFAULT_SCORING, 150, 2, 75.0, 4)
print('decisions', outs[0][0][:6].tolist(), flush=True)
# barcode ranking on the device (top2) over a many-column class, checked against the host ranking of the same records
from porechop_b200 import hostio
from porechop_b200.fastq import Top2Scores, top2_from_scores
cols = list(range(0, len(starts), 7))
(trim, top2, rec), = W.adapter_end_decisions([(sbuf[:150 * 40], soff[:41], a3, o3, True, cols)], wl.DEFAULT_SCORING, 150, 2, 75.0, 4,
                                             want_top2=True, want_records=True)
exp = top2_from_scores(hostio.full_scores(rec.reshape(40, len(starts), 9), cols)) if hostio.LIB is not None else None
got = Top2Scores([str(c) for c in cols], top2).ranked()
ok = exp is None or all(np.array_equal(g, e) for g, e in zip(got, exp))
bad += 0 if ok else 1
print('top2      %s' % ('ok' if ok else 'DIFFERENT'), flush=True)
got = W.adapter_alignment_batch_multi([(sbuf, soff, a1, o1), (lbuf, loff, a2, o2)], wl.DEFAULT_SCORING)
bad += 0 if np.array_equal(got[1], oracle_batch(lbuf, loff, a2, o2, wl.DEFAULT_SCORING)) else 1
# adapter-set search (Phase A): the per-adapter maxima against the host reduction of the oracle's records, over 227 and 2
# adapter columns, with long reads on the two-pass path and with many small chunks
from porechop_b200.align import scores_from_records
for opts in ({}, {'direct_max': 100, 'chunk_tasks': 200}):
    def search():
        batches = [(sbuf[:150 * 40], soff[:41], a3, o3), (lbuf, loff, a2, o2)]
        got = W.adapter_set_search(batches, wl.DEFAULT_SCORING)
        exp = []
        for b, o, a, ao in batches:
            full = scores_from_records(oracle_batch(b, o, a, ao, wl.DEFAULT_SCORING))[0].reshape(len(o) - 1, len(ao) - 1)
            exp.append(np.maximum(full.max(axis=0), 0.0))
        return np.concatenate(got), np.concatenate(exp)
    run('search', opts, search)
# whole-read trimming (adapterTrimReads / adapterTrimReadsDevice): against adapterEndDecisions over host-cut windows +
# adapterMiddleScan over the host-gathered trimmed reads, with one-pass (150) and two-pass (200) windows
from porechop_b200 import fastq                     # noqa: E402
sides = (wl.pack_adapters([yt]) + ([0],), wl.pack_adapters([yb]) + ([0],))
for end_size in (150, 200):
    def trim(device=False):
        if device:
            import torch
            d_buf, d_off = torch.from_numpy(lbuf).cuda(), torch.from_numpy(loff).cuda()
            got = W.adapter_trim_reads_device(d_buf.data_ptr(), d_off.data_ptr(), len(loff) - 1, len(lbuf), -1, sides[0], sides[1],
                                              (a2, o2), wl.DEFAULT_SCORING, end_size, 2, 75.0, 4, 85.0)
        else:
            got = W.adapter_trim_reads(lbuf, loff, sides[0], sides[1], (a2, o2), wl.DEFAULT_SCORING, end_size, 2, 75.0, 4, 85.0)
        (sw, swo), (ew, ewo) = fastq.end_windows(lbuf, loff, end_size)
        (st, sp, _), (et, ep, _) = W.adapter_end_decisions([(sw, swo) + sides[0][:2] + (True, [0]), (ew, ewo) + sides[1][:2] + (False, [0])],
                                                           wl.DEFAULT_SCORING, end_size, 2, 75.0, 4)
        a, b = fastq.trimmed_ranges(np.diff(loff), st, et)
        tb, to = fastq._gather_ranges(lbuf, loff[:-1] + a, loff[:-1] + b)
        n_hits, h = W.adapter_middle_scan(tb, to, a2, o2, wl.DEFAULT_SCORING, 85.0)
        flat = lambda xs: np.concatenate([np.asarray(x, dtype=np.int64).ravel() for x in xs])    # noqa: E731
        return flat(got), flat((st, et, sp, ep, n_hits, h))
    run('trim', {}, trim)
    run('trim_dev', {}, lambda: trim(True))


# output reads cut on the device (adapterTrimSplitReadsDevice): against fastq.emit over adapterTrimReads' decisions
def split_reads():
    import torch
    from porechop_b200 import device_reads
    qual = np.full(len(lbuf), ord('5'), dtype=np.uint8)
    names, name_off = W.pack_sequences(['r%d' % k for k in range(len(loff) - 1)])
    rna = np.zeros(len(loff) - 1, dtype=bool)
    sets = [(('t', yt), ('b', yb))]
    r = device_reads.trim_reads(torch.from_numpy(lbuf).cuda(), torch.from_numpy(loff).cuda(), sets, wl.DEFAULT_SCORING,
                                torch.from_numpy(qual).cuda(), min_split_read_size=100)
    got = fastq.emit_parts(names, name_off, rna, tuple(x.cpu().numpy() for x in r[:5]), 'fastq')
    # the same records formatted on the device (pb200EmitReadsDevice), in both formats
    d_names = [torch.from_numpy(x).cuda() for x in (names, name_off, rna)]
    for fmt in ('fastq', 'fasta'):
        em = device_reads.emit_reads(r, *d_names, fmt)
        parts = tuple(x.cpu().numpy() for x in r[:5])
        if em.data.cpu().numpy().tobytes() != fastq.emit_parts(names, name_off, rna, parts if fmt == 'fastq' else
                                                               (parts[0], None) + parts[2:], fmt):
            return np.zeros(1), np.ones(1)
    # the reads' FASTQ / FASTA bytes parsed on the device (pb200ParseReadsDevice): the host parser's fields
    text = fastq.emit(fastq.FastqBatch(names, name_off, lbuf, loff, qual, loff, rna), fmt='fastq')
    for kind, data in (('fastq', text), ('fasta', fastq.emit(fastq.parse_fastq(text), fmt='fasta'))):
        p = device_reads.parse_reads(torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda(), kind)
        hb = fastq.parse_fastq(data) if kind == 'fastq' else fastq.parse_fasta(data)
        if any(not np.array_equal(x.cpu().numpy(), y) for x, y in zip(p[:5], (hb.name_buf, hb.name_off, hb.seq, hb.seq_off, hb.qual))):
            return np.zeros(1), np.ones(1)
    st, et, _, _, n_hits, h = W.adapter_trim_reads(lbuf, loff, sides[0], sides[1], (a2, o2), wl.DEFAULT_SCORING, 150, 2, 75.0, 4, 85.0)
    middle = fastq.middle_trim_ranges(fastq._hits_dict(n_hits, h), [('t', yt), ('b', yb)], {'t'}, {'b'}, 10, 100)
    batch = fastq.FastqBatch(names, name_off, lbuf, loff, qual, loff, rna)
    exp = fastq.emit(batch, st, et, middle, 'fastq', 100)
    return np.frombuffer(got, dtype=np.uint8), np.frombuffer(exp, dtype=np.uint8)


run('split_dev', {}, split_reads)


# demultiplexed output reads (adapterDemuxReadsDevice): each bin's bytes against fastq.demux_fastq, over 12 barcode sets
def demux_reads():
    import torch
    from porechop_b200 import device_reads
    bs, be = wl.demux_adapters()
    buf, off = wl.synth_reads(8, bs[3] + yt, yb + be[3], seed=3, chimera_p=0.5, max_len=4000)
    qual = np.full(len(buf), ord('5'), dtype=np.uint8)
    n = len(off) - 1
    names, name_off = W.pack_sequences(['r%d' % k for k in range(n)])
    batch = fastq.FastqBatch(names, name_off, buf, off, qual, off, np.zeros(n, dtype=bool))
    sets = [('Y', ('t', yt), ('b', yb))] + [('Barcode %d (forward)' % (j + 1), ('BC%02d' % (j + 1), bs[j]),
                                             ('BC%02d_end' % (j + 1), be[j])) for j in range(12)]
    bc = dict(forward_or_reverse='forward', barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=False,
              discard_unassigned=False)
    r = device_reads.demux_reads(torch.from_numpy(buf).cuda(), torch.from_numpy(off).cuda(), sets, wl.DEFAULT_SCORING,
                                 torch.from_numpy(qual).cuda(), min_split_read_size=100, **bc)
    parts = tuple(x.cpu().numpy() for x in r[:5])
    em = device_reads.emit_reads(r, *(torch.from_numpy(x).cuda() for x in (names, name_off, batch.rna)), 'fastq')
    data = em.data.cpu().numpy().tobytes()
    got = b''.join(data[b0:b1] for b0, b1 in em.bins.values())
    assert got == b''.join(fastq.emit_parts(names, name_off, batch.rna, parts[:2] + (parts[2][r0:r1 + 1], parts[3][r0:r1],
                                                                            parts[4][r0:r1]), 'fastq') for r0, r1 in r.bins.values())
    bins, _ = fastq.demux_fastq(batch, sets, wl.DEFAULT_SCORING, min_split_read_size=100, **bc)
    exp = b''.join(bins[k] for k in r.bins) if sorted(bins) == sorted(r.bins) else b''
    return np.frombuffer(got, dtype=np.uint8), np.frombuffer(exp, dtype=np.uint8)


run('demux_dev', {}, demux_reads)
print('SANITIZE RUN COMPLETE, %d wrong' % bad, flush=True)
sys.exit(1 if bad else 0)
