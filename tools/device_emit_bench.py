"""Porechop's output files for records in GPU memory: two ways to get the bytes, alternated in one run over the same records.

    python tools/device_emit_bench.py [--reads 200000] [--repeats 3] [--out results/device_emit_bench.json]
    python tools/device_emit_bench.py --profile SHAPE [--reads 200000]      (kernel times of one shape, 0 .. 4, in a run of its own)

  (a) every record (bases, qualities, offsets, read, part) is copied home, then each bin is fastq.emit_parts over its slice
      (device_demux_bench.py path (b)); one file for trim_reads -- what a caller had to do before pb200EmitReadsDevice;
  (b) device_reads.emit_reads formats the records on the device (the names uploaded first), then the bytes come home in one
      copy into pinned memory and each bin is a slice (a view) of it, which a caller writes to its file as it is.

Shapes over the config-4 read model with barcodes (device_demux_bench.reads: 8-kb log-normal lengths, 5 % chimeras, random
qualities), resident in GPU memory: one file (trim_reads) in FASTQ, in FASTA, and in FASTQ with 20 % of the reads flagged RNA;
48 and 96 bins (demux_reads) in FASTQ.  Per repeat the device call that makes the records runs once and the two paths format
its records in alternating order.  Reports medians of the repeats (host clock around work that ends in a device synchronise):
the records' call, (a) copy home and emit_parts, (b) names upload, emit_reads, copy home and slicing; the PCIe bytes computed
from the shapes; and whether both paths give byte-identical bins.  --profile takes the emit kernels of one shape from
torch.profiler in a process of its own (one profiler session per process), with the write kernel's bytes per second next to
a same-size device-to-device copy in the same run.  The card's name, power limit and SM clock are read in the same run.  Needs a CUDA device; there is no CPU fallback.
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

from device_demux_bench import reads  # noqa: E402
from device_output_bench import gpu_conditions  # noqa: E402

DEFAULT = (3, -6, -5, -2)
SHAPES = [('trim', 48, 'fastq', 0.0), ('trim', 48, 'fasta', 0.0), ('trim', 48, 'fastq', 0.2), ('demux', 48, 'fastq', 0.0),
          ('demux', 96, 'fastq', 0.0)]


def run(n_reads, kind, k, fmt, rna_share, repeats, profile_only=False):
    import torch
    from porechop_b200 import device_reads, fastq
    assert torch.cuda.is_available(), 'this benchmark needs a CUDA device'
    buf, off, qual, names, name_off, rna, sets = reads(n_reads, k)
    rna = np.random.default_rng(2).random(n_reads) < rna_share
    d_seq, d_qual, d_off = (torch.from_numpy(x).cuda() for x in (buf, qual, off))
    opts = dict(min_split_read_size=1000)
    bc = dict(forward_or_reverse='forward', barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=False)

    def call():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if kind == 'trim':
            r = device_reads.trim_reads(d_seq, d_off, sets, DEFAULT, d_qual if fmt == 'fastq' else None, **opts)
        else:
            r = device_reads.demux_reads(d_seq, d_off, sets, DEFAULT, d_qual if fmt == 'fastq' else None,
                                         discard_unassigned=False, **bc, **opts)
        torch.cuda.synchronize()
        return r, time.perf_counter() - t0

    def ranges(r):
        return r.bins if kind == 'demux' else {'out': (0, len(r.read))}

    def path_a(r):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        parts = tuple(x.cpu().numpy() if x is not None else None for x in r[:5])
        t1 = time.perf_counter()
        bins = {nm: fastq.emit_parts(names, name_off, rna, parts[:2] + (parts[2][r0:r1 + 1], parts[3][r0:r1], parts[4][r0:r1]),
                                     fmt) for nm, (r0, r1) in ranges(r).items()}
        t2 = time.perf_counter()
        return bins, {'copy_home': t1 - t0, 'emit_parts': t2 - t1, 'total': t2 - t0}

    def path_b(r):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        d_names, d_name_off, d_rna = (torch.from_numpy(x).cuda() for x in (names, name_off, rna))
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        em = device_reads.emit_reads(r, d_names, d_name_off, d_rna, fmt)
        t2 = time.perf_counter()
        host = torch.empty(em.data.numel(), dtype=torch.uint8, pin_memory=True)
        host.copy_(em.data)
        data = host.numpy()
        t3 = time.perf_counter()
        bins = {nm: data[b0:b1] for nm, (b0, b1) in (em.bins or {'out': (0, len(data))}).items()}
        t4 = time.perf_counter()
        return bins, {'upload_names': t1 - t0, 'emit': t2 - t1, 'copy_home': t3 - t2, 'slices': t4 - t3, 'total': t4 - t0}, em

    shape = '%s %s%s%s' % (kind, fmt, ' %d bins' % k if kind == 'demux' else '', ' %d%% RNA' % round(100 * rna_share) if rna_share else '')
    r, _ = call()                     # warm-up (module load, engine buffers, pinned staging), then the identity check
    if profile_only:
        return kernel_profile(r, shape, names, name_off, rna, fmt)
    bins_a, _ = path_a(r)
    bins_b, _, em = path_b(r)
    same = sorted(bins_a) == sorted(bins_b) and all(np.array_equal(np.frombuffer(bins_a[x], dtype=np.uint8), bins_b[x]) for x in bins_a)
    times = {'call': [], 'a': [], 'b': []}
    for i in range(repeats):
        r, t = call()
        times['call'].append(t)
        for p in ('ab' if i % 2 == 0 else 'ba'):
            times[p].append(path_a(r)[1] if p == 'a' else path_b(r)[1])
    n_rec, n_bases, n_out = len(r.read), len(r.seq), int(em.data.numel())
    n_bins = len(ranges(r))
    qual_bytes = n_bases if fmt == 'fastq' else 0
    pcie = {'a': n_bases + qual_bytes + 8 * (n_rec + 1) + 8 * n_rec,            # bases, qualities, offsets, read + part home
            'b': len(names) + 8 * (n_reads + 1) + n_reads                     # names, offsets and RNA flags up
                 + 8 * (n_reads + 1) + 8 + n_out                              # name offsets (the size bound), total, output home
                 + (8 * (n_rec + 1) if kind == 'demux' else 0)}               # record offsets home (bin byte ranges)
    med = lambda xs: float(np.median(xs))                   # noqa: E731
    return {
        'shape': shape, 'reads': n_reads, 'bases': int(len(buf)), 'records': n_rec, 'record_bases': n_bases, 'out_bytes': n_out,
        'bins_with_records': n_bins, 'identical_bins': bool(same), 'repeats': repeats,
        'call_seconds': med(times['call']),
        'a_seconds': {x: med([t[x] for t in times['a']]) for x in times['a'][0]},
        'b_seconds': {x: med([t[x] for t in times['b']]) for x in times['b'][0]},
        'a_total_all': [t['total'] for t in times['a']], 'b_total_all': [t['total'] for t in times['b']],
        'pcie_bytes': pcie,
    }


def kernel_profile(r, shape, names, name_off, rna, fmt):
    """the emit kernels of one emit_reads call (after a warm-up call), and a same-size device-to-device copy"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from porechop_b200 import device_reads
    device_reads.emit_reads(r, torch.from_numpy(names).cuda(), torch.from_numpy(name_off).cuda(), torch.from_numpy(rna).cuda(), fmt)
    d_names, d_name_off, d_rna = (torch.from_numpy(x).cuda() for x in (names, name_off, rna))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        em = device_reads.emit_reads(r, d_names, d_name_off, d_rna, fmt)
    kern = {}
    for ev in prof.key_averages():
        us = getattr(ev, 'self_device_time_total', None)
        if us is None:
            us = getattr(ev, 'self_cuda_time_total', 0)
        if us > 0:
            kern[ev.key] = kern.get(ev.key, 0.0) + us / 1000.0      # ms
    write_ms = sum(v for x, v in kern.items() if 'emit_write_kernel' in x)
    count_ms = sum(v for x, v in kern.items() if 'emit_count_kernel' in x)
    scan_ms = sum(v for x, v in kern.items() if 'scan_' in x)
    n_rec, n_bases, n_out = len(r.read), len(r.seq), int(em.data.numel())
    name_bytes = int((np.diff(name_off)[r.read.cpu().numpy()]).sum())
    # the write kernel reads the records' bases (and qualities), their names and 41 B of per-record arrays, and writes the output
    moved = n_bases * (2 if fmt == 'fastq' else 1) + name_bytes + 41 * n_rec + n_out
    src = torch.empty(n_out, dtype=torch.uint8, device='cuda')
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    e0.record()
    for _ in range(reps):
        dst.copy_(src)
    e1.record()
    torch.cuda.synchronize()
    memcpy_ms = e0.elapsed_time(e1) / reps

    return {
        'shape': shape, 'out_bytes': n_out,
        'profile_ms': {'emit_count_kernel': count_ms, 'scan': scan_ms, 'emit_write_kernel': write_ms},
        'write_kernel_TBps': moved / (write_ms * 1e-3) / 1e12 if write_ms else None,
        'memcpy_d2d_TBps': 2 * n_out / (memcpy_ms * 1e-3) / 1e12, 'write_kernel_bytes': moved,
    }


if __name__ == '__main__':
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--reads', type=int, default=200000)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default='')
    ap.add_argument('--profile', type=int, default=None, help='index into SHAPES: only the kernel times of that shape')
    a = ap.parse_args()
    import torch
    res = {'gpu': gpu_conditions(), 'torch_device': torch.cuda.get_device_name(0), 'runs': []}
    for shape in SHAPES if a.profile is None else [SHAPES[a.profile]]:
        res['runs'].append(run(a.reads, *shape, a.repeats, profile_only=a.profile is not None))
        print(json.dumps(res['runs'][-1]), flush=True)
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    assert all(r.get('identical_bins', True) for r in res['runs']), 'the two paths gave different bins'
