"""FASTQ / FASTA parsing and whole chunks from input bytes to output bytes: the host path against the device path, alternated in one
run over the same bytes.

    python tools/device_parse_bench.py [--chunk-mb 256] [--repeats 3] [--out results/device_parse_bench.json]
    python tools/device_parse_bench.py --profile INPUT [--chunk-mb 256]      (parse kernel times of one input, 0 or 1, on their own)

Inputs: the config-4 read model (workloads.synth_reads_fast: 8-kb log-normal lengths, 5 % chimeras, random qualities, names with
spaces) as FASTQ bytes of the flat CLI's chunk size (256 MB), and the same reads as 70-column FASTA.
  parse:  (a) fastq.parse_fastq / parse_fasta, then the bases, qualities and names (with their offsets) uploaded -- what a
              caller of trim_reads did so far; (b) the raw bytes uploaded through pinned memory, then device_reads.parse_reads.
  chunk:  (a) fastq.trim_fastq with PB200_DEVICE_DECISIONS and PB200_DEVICE_MIDDLE on (host parse, one adapterTrimReads call,
              host emit); (b) device_reads.trim_fastq (upload, parse, trim and split, emit on the device, one copy home).
Reports medians of the repeats (host clock around work that ends in a device synchronise), input GB/s, the PCIe bytes computed
from the shapes, and whether the two paths give identical fields / bytes.  The card's name, power limit and SM clock are read in
the same run.  --profile takes the parse kernels from torch.profiler in a process of its own (one profiler session per process).
Needs a CUDA device; there is no CPU fallback.
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
INPUTS = ['fastq', 'fasta']


def chunk_bytes(chunk_mb, kind):
    """config-4 reads as FASTQ bytes of about chunk_mb MB (whole records), or the same reads as 70-column FASTA"""
    from porechop_b200 import cpp_function_wrappers as W, fastq, workloads as wl
    yt, yb = wl.nsk007()
    n = max(1, int(chunk_mb * (1 << 20) / (2 * 8040 + 40)))
    buf, off = wl.synth_reads_fast(n, yt, yb, chimera_p=0.05)
    qual = np.random.default_rng(1).integers(33, 75, len(buf), dtype=np.uint8)
    names, name_off = W.pack_sequences(['r%d runid=ab ch=%d' % (k, k % 512) for k in range(n)])
    batch = fastq.FastqBatch(names, name_off, buf, off, qual, off.copy(), np.zeros(n, dtype=bool))
    return fastq.emit(batch, fmt=kind), [(('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))]


def run(chunk_mb, kind, repeats):
    import torch
    from porechop_b200 import device_reads, fastq
    assert torch.cuda.is_available(), 'this benchmark needs a CUDA device'
    data, sets = chunk_bytes(chunk_mb, kind)
    host_parse = fastq.parse_fastq if kind == 'fastq' else fastq.parse_fasta

    def parse_a():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        b = host_parse(data)
        t1 = time.perf_counter()
        up = [torch.from_numpy(x).cuda() for x in (b.name_buf, b.name_off, b.seq, b.seq_off, b.qual)]
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        return (b, up), {'parse': t1 - t0, 'upload': t2 - t1, 'total': t2 - t0}

    def parse_b():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        d = device_reads.device().upload_bytes(data)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        p = device_reads.parse_reads(d, kind)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        return p, {'upload': t1 - t0, 'parse': t2 - t1, 'total': t2 - t0}

    def chunk_a():
        fastq.DEVICE_DECISIONS = fastq.DEVICE_MIDDLE = True
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out, _ = fastq.trim_fastq(host_parse(data), sets, DEFAULT, fmt=kind, as_array=True)
        return out, {'total': time.perf_counter() - t0}

    def chunk_b():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out, _ = device_reads.trim_fastq(data, sets, DEFAULT, fmt=kind, as_array=True, kind=kind)
        return out, {'total': time.perf_counter() - t0}

    # warm-up and identity checks
    (b, _), _ = parse_a()
    p, _ = parse_b()
    same_parse = all(np.array_equal(x.cpu().numpy(), y) for x, y in zip(
        (p.names, p.name_off, p.seq, p.seq_off, p.qual), (b.name_buf, b.name_off, b.seq, b.seq_off, b.qual))) and \
        np.array_equal(p.rna.cpu().numpy().astype(bool), b.rna)
    same_chunk = np.array_equal(np.asarray(chunk_a()[0]), np.asarray(chunk_b()[0]))
    out_bytes = len(chunk_b()[0])
    del p
    times = {k: [] for k in ('parse_a', 'parse_b', 'chunk_a', 'chunk_b')}
    fns = {'parse_a': parse_a, 'parse_b': parse_b, 'chunk_a': chunk_a, 'chunk_b': chunk_b}
    for i in range(repeats):
        for k in (('parse_a', 'parse_b', 'chunk_a', 'chunk_b') if i % 2 == 0 else ('parse_b', 'parse_a', 'chunk_b', 'chunk_a')):
            times[k].append(fns[k]()[1])
    n, n_in, n_seq, n_names = len(b), len(data), len(b.seq), len(b.name_buf)
    med = lambda ts: {x: float(np.median([t[x] for t in ts])) for x in ts[0]}      # noqa: E731
    res = {'input': kind, 'reads': n, 'input_bytes': n_in, 'bases': n_seq, 'output_bytes': out_bytes, 'repeats': repeats,
           'identical_parse': bool(same_parse), 'identical_output': bool(same_chunk)}
    for k in times:
        res[k + '_seconds'] = med(times[k])
        res[k + '_input_GBps'] = n_in / res[k + '_seconds']['total'] / 1e9
    res['pcie_bytes'] = {
        'parse_a': n_names + n_seq * 2 + 16 * (n + 1),                     # names, bases, qualities and two offset arrays up
        'parse_b': n_in + 8 * 4,                                          # the raw bytes up; line count and totals home
        'chunk_a': n_seq + 8 * (n + 1),                                   # the bases and offsets up (decisions home are small)
        'chunk_b': n_in + 8 * (n + 1) + out_bytes,                        # raw bytes up, name offsets (emit's bound) and output home
    }
    return res


def kernel_profile(chunk_mb, kind):
    """the kernels of one parse_reads call (after a warm-up call)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from porechop_b200 import device_reads
    data, _ = chunk_bytes(chunk_mb, kind)
    d = device_reads.device().upload_bytes(data)
    device_reads.parse_reads(d, kind)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        device_reads.parse_reads(d, kind)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        us = getattr(ev, 'self_device_time_total', None)
        if us is None:
            us = getattr(ev, 'self_cuda_time_total', 0)
        if us > 0 and ('parse_' in ev.key or 'scan_' in ev.key or 'Memcpy' in ev.key or 'Memset' in ev.key):
            kern[ev.key.split('(')[0]] = kern.get(ev.key.split('(')[0], 0.0) + us / 1000.0      # ms
    total = sum(v for x, v in kern.items() if 'parse_' in x or 'scan_' in x)
    return {'input': kind, 'input_bytes': len(data), 'profile_ms': kern, 'kernels_ms': total,
            'kernels_input_GBps': len(data) / (total * 1e-3) / 1e9 if total else None}


if __name__ == '__main__':
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--chunk-mb', type=float, default=256)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default='')
    ap.add_argument('--profile', type=int, default=None, help='index into INPUTS: only the parse kernel times of that input')
    a = ap.parse_args()
    import torch
    res = {'gpu': gpu_conditions(), 'torch_device': torch.cuda.get_device_name(0), 'runs': []}
    for kind in INPUTS if a.profile is None else [INPUTS[a.profile]]:
        res['runs'].append(run(a.chunk_mb, kind, a.repeats) if a.profile is None else kernel_profile(a.chunk_mb, kind))
        print(json.dumps(res['runs'][-1]), flush=True)
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    assert all(r.get('identical_parse', True) and r.get('identical_output', True) for r in res['runs']), \
        'the two paths gave different results'
