"""Demultiplexed output reads for device-resident reads: two ways to get each bin's file, alternated in one run.

    python tools/device_demux_bench.py [--reads 200000] [--bins 48 96] [--repeats 3] [--out results/device_demux_bench.json]

  (a) device_reads.trim_reads(barcodes=...): the records come back in read order with one bin name per read (the ranking comes
      home and is called on the host); every record is copied home, and each bin is emit_parts(select=calls == name) --
      what a caller had to do before adapterDemuxReadsDevice;
  (b) device_reads.demux_reads: the bins are called on the device and the records come back grouped by bin; each bin's slice
      of records is copied home and written by emit_parts.

Reads: the config-4 read model (workloads.synth_reads_fast: 8-kb log-normal lengths, 5 % chimeras) with a barcode before the Y
adapters -- 8 blocks of reads, each with one of the barcodes spread over the bins -- and random qualities, resident in GPU
memory.  Adapter sets: {Y_Top, Y_Bottom} and the first 48 / 96 sequences of workloads.demux_adapters() as BCnn sets.  Reports
per path the median of the repeats of the whole path and of the device call alone (host clock around work that ends in a
device synchronise), the PCIe bytes computed from the shapes, and whether both paths give byte-identical bins; in a separate
run the demux stage's kernels and the gather from torch.profiler.  The card's name, power limit and SM clock are read in the
same run.  Needs a CUDA device; there is no CPU fallback.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from device_output_bench import gpu_conditions  # noqa: E402

DEFAULT = (3, -6, -5, -2)
DEMUX_KERNELS = ('barcode_call_kernel', 'demux_count_kernel', 'demux_bin_parts_kernel', 'demux_scatter_kernel')


def reads(n_reads, k):
    from porechop_b200 import cpp_function_wrappers as W, workloads as wl
    yt, yb = wl.nsk007()
    bs, be = wl.demux_adapters()
    blocks = 8
    per = [n_reads // blocks + (1 if b < n_reads % blocks else 0) for b in range(blocks)]
    bufs, offs, base = [], [np.zeros(1, dtype=np.int64)], 0
    for b in range(blocks):
        j = (b * k) // blocks
        buf, off = wl.synth_reads_fast(per[b], bs[j] + yt, yb + be[j], chimera_p=0.05)
        bufs.append(buf)
        offs.append(np.asarray(off[1:], dtype=np.int64) + base)
        base += len(buf)
    buf, off = np.concatenate(bufs), np.concatenate(offs)
    qual = np.random.default_rng(1).integers(33, 75, len(buf), dtype=np.uint8)
    names, name_off = W.pack_sequences(['r%d' % i for i in range(n_reads)])
    sets = [('SQK-NSK007', ('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))] + \
           [('Barcode %d (forward)' % (j + 1), ('BC%02d' % (j + 1), bs[j]), ('BC%02d_end' % (j + 1), be[j])) for j in range(k)]
    return buf, off, qual, names, name_off, np.zeros(n_reads, dtype=bool), sets


def run(n_reads, k, repeats):
    import torch
    from porechop_b200 import device_reads, fastq
    assert torch.cuda.is_available(), 'this benchmark needs a CUDA device'
    buf, off, qual, names, name_off, rna, sets = reads(n_reads, k)
    d_seq, d_qual, d_off = (torch.from_numpy(x).cuda() for x in (buf, qual, off))
    opts = dict(min_split_read_size=1000)
    bc = dict(forward_or_reverse='forward', barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=False)

    def path_a():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = device_reads.trim_reads(d_seq, d_off, sets, DEFAULT, d_qual, barcodes=bc, **opts)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        parts = tuple(x.cpu().numpy() for x in r[:5])
        calls = np.array(r.calls, dtype=object)
        bins = {}
        for name in dict.fromkeys(r.calls):
            out = fastq.emit_parts(names, name_off, rna, parts, 'fastq', select=(calls == name))
            if len(out):
                bins[name] = out
        t2 = time.perf_counter()
        return bins, r, {'call': t1 - t0, 'total': t2 - t0}

    def path_b():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = device_reads.demux_reads(d_seq, d_off, sets, DEFAULT, d_qual, discard_unassigned=False, **bc, **opts)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        bins = {}
        for name, (r0, r1) in r.bins.items():
            o = r.off[r0:r1 + 1].cpu().numpy()
            b0, b1 = int(o[0]), int(o[-1])
            parts = (r.seq[b0:b1].cpu().numpy(), r.qual[b0:b1].cpu().numpy(), o - b0, r.read[r0:r1].cpu().numpy(),
                     r.part[r0:r1].cpu().numpy())
            bins[name] = fastq.emit_parts(names, name_off, rna, parts, 'fastq')
        t2 = time.perf_counter()
        return bins, r, {'call': t1 - t0, 'total': t2 - t0}

    # warm-up (module load, engine buffers), then the identity check at the timed size
    bins_a, ra, _ = path_a()
    bins_b, rb, _ = path_b()
    same = sorted(bins_a) == sorted(bins_b) and all(bins_a[x] == bins_b[x] for x in bins_a) and ra.calls == rb.calls
    times = {'a': [], 'b': []}
    for _ in range(repeats):
        times['a'].append(path_a()[2])
        times['b'].append(path_b()[2])

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        path_b()
    kern = {}
    for ev in prof.key_averages():
        us = getattr(ev, 'self_device_time_total', None)
        if us is None:
            us = getattr(ev, 'self_cuda_time_total', 0)
        if us > 0:
            kern[ev.key] = kern.get(ev.key, 0.0) + us / 1000.0      # ms
    demux_ms = {d: sum(v for x, v in kern.items() if d in x) for d in DEMUX_KERNELS}
    gather_ms = sum(v for x, v in kern.items() if 'split_gather_kernel' in x)
    total_kernel_ms = sum(v for x, v in kern.items() if 'Memcpy' not in x and 'Memset' not in x)

    n_parts, n_out, n_hits = len(rb.read), len(rb.seq), sum(len(v) for v in rb.hits.values())
    _, _, su, eu = fastq.barcode_columns(fastq._norm_sets(sets), 'forward')
    n_bins = len(dict.fromkeys(su + eu))
    decisions = n_reads * 4 * 3 + n_hits * (40 + 16)          # two trims and n_hits per read; hit records home, hit CSR up
    records = 2 * n_out + 8 * n_parts + 4 * n_parts * 2       # bases, qualities, offsets, read and part of every record
    pcie = {'a': decisions + n_reads * 2 * 24 + records + 8,  # + both sides' top-2 ranking home
            'b': decisions + n_reads * 4 + 8 * (n_bins + 2) + records + 8 * len(rb.bins)}   # + read bins, bin offsets
    med = lambda xs: float(np.median(xs))                   # noqa: E731
    return {
        'bins_named': n_bins, 'bins_with_records': len(rb.bins), 'reads': n_reads, 'bases': int(len(buf)),
        'records': n_parts, 'out_bases': n_out, 'hits': n_hits, 'identical_bins': bool(same), 'repeats': repeats,
        'a_seconds': {x: med([t[x] for t in times['a']]) for x in ('call', 'total')},
        'b_seconds': {x: med([t[x] for t in times['b']]) for x in ('call', 'total')},
        'a_total_all': [t['total'] for t in times['a']], 'b_total_all': [t['total'] for t in times['b']],
        'profile_ms': dict(demux_ms, split_gather_kernel=gather_ms, all_kernels=total_kernel_ms),
        'pcie_bytes': pcie,
    }


if __name__ == '__main__':
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--reads', type=int, default=200000)
    ap.add_argument('--bins', type=int, nargs='+', default=[48, 96])
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default='')
    a = ap.parse_args()
    import torch
    res = {'gpu': gpu_conditions(), 'torch_device': torch.cuda.get_device_name(0),
           'runs': [run(a.reads, k, a.repeats) for k in a.bins]}
    print(json.dumps(res, indent=1))
    assert all(r['identical_bins'] for r in res['runs']), 'the two paths gave different bins'
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
