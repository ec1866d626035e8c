"""gzip of Porechop's output on the device (device_reads.gzip_bytes, pb200GzipDevice) against the host's block-parallel zlib
(hostio.gzip_members), alternated in one run over the same bytes.

    python tools/device_gzip_bench.py [--chunk-mb 256] [--repeats 3] [--out results/device_gzip_bench.json]
    python tools/device_gzip_bench.py --profile [--chunk-mb 256]      (kernel times, in a run of its own)

Input: the config-4 read model (device_parse_bench.chunk_bytes: 8-kb log-normal reads, 5 % chimeras) with qualities as runs
(geometric lengths) of a random walk over Phred 2..40 -- uniform random qualities would misstate every ratio.  Shapes, the
output bytes already in GPU memory: one FASTQ file, one FASTA file, and the FASTQ bytes as 48 bins (48 segments cut at record
boundaries: each bin is its own .gz).
  (a) the bytes come home into pinned memory, then hostio.gzip_members compresses each bin at level 6 (a6) and at level 1 (a1)
      on every CPU the process may use (4 MB members, OpenMP);
  (b) gzip_bytes compresses each bin on the device, and the compressed bytes come home into pinned memory.
Whole chunk (FASTQ, chunk-mb of input): device_reads.trim_fastq(gz=True) against device_reads.trim_fastq + gzip_members at level
6 and 1.  Medians of the repeats (host clock around work that ends in a device synchronise), GB/s of uncompressed bytes,
compressed sizes and ratios, the PCIe bytes of each path computed from the sizes, and whether every output decompresses to the
input.  The card's name, power limit and SM clock are read in the same run.  Needs a CUDA device; there is no CPU fallback.
"""
import argparse
import json
import os
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from device_output_bench import gpu_conditions  # noqa: E402

DEFAULT = (3, -6, -5, -2)


def chunk(chunk_mb, kind, seed=1):
    """config-4 reads with run-structured qualities as FASTQ / FASTA bytes, and their adapter sets"""
    from porechop_b200 import cpp_function_wrappers as W, fastq, workloads as wl
    yt, yb = wl.nsk007()
    n = max(1, int(chunk_mb * (1 << 20) / (2 * 8040 + 40)))
    buf, off = wl.synth_reads_fast(n, yt, yb, chimera_p=0.05)
    rng = np.random.default_rng(seed)
    walk = np.abs(((np.cumsum(rng.integers(-4, 5, len(buf))) + 20) % 76) - 38) + 2
    qual = np.repeat(walk, rng.geometric(0.35, len(buf)))[:len(buf)].astype(np.uint8) + 33
    names, name_off = W.pack_sequences(['%032x runid=ab read=%d ch=%d' % (int(rng.integers(0, 1 << 62)) << 64 | k, k, k % 512)
                                        for k in range(n)])
    batch = fastq.FastqBatch(names, name_off, buf, off, qual, off.copy(), np.zeros(n, dtype=bool))
    return fastq.emit(batch, fmt=kind), [(('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))]


def bins_of(data, k):
    """k ranges of data cut at record starts ('\\n@' of FASTQ)"""
    starts = [0]
    for j in range(1, k):
        p = data.find(b'\n@', j * len(data) // k)
        starts.append(p + 1 if p >= 0 else len(data))
    starts.append(len(data))
    return {'bin%02d' % j: (starts[j], starts[j + 1]) for j in range(k)}


def _inflate_all(blob):
    """the decompression of a multi-member .gz, fed in 1 MB pieces (linear in the number of members)"""
    blob, out, pos = bytes(blob), [], 0
    while pos < len(blob):
        d = zlib.decompressobj(31)
        while not d.eof and pos < len(blob):
            piece = blob[pos:pos + (1 << 20)]
            out.append(d.decompress(piece))
            pos += len(piece)
        pos -= len(d.unused_data)
    return b''.join(out)


def run(chunk_mb, repeats):
    import torch
    from porechop_b200 import device_reads, hostio
    assert torch.cuda.is_available(), 'this benchmark needs a CUDA device'
    fq, sets = chunk(chunk_mb, 'fastq')
    fa, _ = chunk(chunk_mb, 'fasta')
    shapes = {'fastq_file': (fq, None), 'fasta_file': (fa, None), 'fastq_48_bins': (fq, bins_of(fq, 48))}
    res = {'gpu': gpu_conditions(), 'cpus': len(os.sched_getaffinity(0)), 'chunk_mb': chunk_mb, 'repeats': repeats,
           'quality_model': 'runs (geometric, p = 0.35) of a random walk over Phred 2..40', 'shapes': {}}
    for name, (data, ranges) in shapes.items():
        d = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()
        pinned = torch.empty(len(data), dtype=torch.uint8, pin_memory=True)
        spans = ranges or {'all': (0, len(data))}

        def host(level):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pinned.copy_(d)
            h = pinned.numpy()
            out = {k: hostio.gzip_members(h[b0:b1], level=level) for k, (b0, b1) in spans.items()}
            return out, time.perf_counter() - t0

        def dev():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            g = device_reads.gzip_bytes(d, ranges)
            h = torch.empty(g.data.numel(), dtype=torch.uint8, pin_memory=True)
            h.copy_(g.data)
            hn = h.numpy()
            out = {k: hn[b0:b1] for k, (b0, b1) in (g.ranges or {'all': (0, len(hn))}).items()}
            return out, time.perf_counter() - t0

        fns = {'a6': lambda: host(6), 'a1': lambda: host(1), 'b': dev}
        sizes, ok = {}, {}
        for k, f in fns.items():                                     # warm-up, sizes and round trips
            out, _ = f()
            sizes[k] = int(sum(len(v) for v in out.values()))
            ok[k] = all(_inflate_all(out[n]) == data[b0:b1] for n, (b0, b1) in spans.items())
        times = {k: [] for k in fns}
        order = list(fns)
        for i in range(repeats):
            for k in (order if i % 2 == 0 else order[::-1]):
                times[k].append(fns[k]()[1])
        r = {'input_bytes': len(data), 'bins': len(spans), 'round_trip_ok': ok, 'compressed_bytes': sizes,
             'ratio': {k: len(data) / v for k, v in sizes.items()}}
        r['seconds'] = {k: float(np.median(v)) for k, v in times.items()}
        r['input_GBps'] = {k: len(data) / v / 1e9 for k, v in r['seconds'].items()}
        r['pcie_bytes_home'] = {'a6': len(data), 'a1': len(data), 'b': sizes['b']}
        res['shapes'][name] = r
        print('shape %s: %s' % (name, json.dumps(r['seconds'])), file=sys.stderr, flush=True)
        del d, pinned
        torch.cuda.empty_cache()

    # whole chunk: input bytes to .gz bytes
    def whole(level):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if level is None:
            out, _ = device_reads.trim_fastq(fq, sets, DEFAULT, as_array=True, gz=True)
        else:
            plain, _ = device_reads.trim_fastq(fq, sets, DEFAULT, as_array=True)
            out = hostio.gzip_members(plain, level=level)
        return out, time.perf_counter() - t0
    fns = {'device_gzip': lambda: whole(None), 'host_level6': lambda: whole(6), 'host_level1': lambda: whole(1)}
    plain, _ = device_reads.trim_fastq(fq, sets, DEFAULT, as_array=True)
    sizes, ok = {}, {}
    for k, f in fns.items():
        out, _ = f()
        sizes[k], ok[k] = len(out), _inflate_all(out) == plain.tobytes()
    times = {k: [] for k in fns}
    for i in range(repeats):
        for k in (list(fns) if i % 2 == 0 else list(fns)[::-1]):
            times[k].append(fns[k]()[1])
    res['whole_chunk'] = {'input_bytes': len(fq), 'output_bytes': int(len(plain)), 'round_trip_ok': ok, 'compressed_bytes': sizes,
                          'seconds': {k: float(np.median(v)) for k, v in times.items()},
                          'input_GBps': {k: len(fq) / float(np.median(v)) / 1e9 for k, v in times.items()}}
    return res


def kernel_profile(chunk_mb):
    """the gzip call's kernels from torch.profiler, next to a same-size device-to-device copy"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from porechop_b200 import device_reads
    fq, _ = chunk(chunk_mb, 'fastq')
    d = torch.from_numpy(np.frombuffer(fq, dtype=np.uint8).copy()).cuda()
    dst = torch.empty_like(d)
    device_reads.gzip_bytes(d)
    dst.copy_(d)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            device_reads.gzip_bytes(d)
            dst.copy_(d)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_time_total > 0:
            out[e.key] = {'calls': e.count, 'us_per_call': e.device_time_total / max(e.count, 1)}
    return {'gpu': gpu_conditions(), 'input_bytes': len(fq), 'kernels': out}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--chunk-mb', type=float, default=256)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default='')
    ap.add_argument('--profile', action='store_true')
    a = ap.parse_args()
    res = kernel_profile(a.chunk_mb) if a.profile else run(a.chunk_mb, a.repeats)
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(text + '\n')


if __name__ == '__main__':
    main()
