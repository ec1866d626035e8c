"""Porechop's output reads for device-resident reads: two ways to get them, alternated in one run.

    python tools/device_output_bench.py [--reads 200000] [--repeats 3] [--out results/device_output_bench.json]

  (a) adapterTrimReadsDevice (trims and hits come home), then the reads and qualities copied home into pinned memory and cut by
      fastq.emit's host logic -- what a caller with reads in GPU memory had to do before adapterTrimSplitReadsDevice;
  (b) adapterTrimSplitReadsDevice through device_reads.trim_reads: the records are cut on the device and stay there.

Reads: the config-4 read model (workloads.synth_reads_fast: 8-kb log-normal lengths, 5 % chimeras, {Y_Top, Y_Bottom}) with
random qualities, resident in GPU memory.  Reports the time of each path (host clock around work that ends in a device
synchronise), the output stage's kernels from torch.profiler in a separate run, the gather kernel's bytes moved per second next
to a same-size device-to-device copy measured in the same run and the 3.35 TB/s data-sheet figure, the PCIe bytes of each path
computed from the shapes, and whether both paths give the same output bytes.  The card's name, power limit and SM clock are
read in the same run.  Needs a CUDA device; there is no CPU fallback.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULT = (3, -6, -5, -2)
HBM_TBPS = 3.35                    # H100 SXM data sheet, HBM3


def gpu_conditions():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(','), [x.strip() for x in out[0].split(',')])) if out else {}
    except (OSError, subprocess.SubprocessError):
        return {}


def run(n_reads, repeats, out_path):
    import torch
    from porechop_b200 import cpp_function_wrappers as W, device_reads, fastq, workloads as wl
    assert torch.cuda.is_available(), 'this benchmark needs a CUDA device'
    yt, yb = wl.nsk007()
    buf, off = wl.synth_reads_fast(n_reads, yt, yb, chimera_p=0.05)
    qual = np.random.default_rng(1).integers(33, 75, len(buf), dtype=np.uint8)
    names, name_off = W.pack_sequences(['r%d' % k for k in range(n_reads)])
    rna = np.zeros(n_reads, dtype=bool)
    d_seq, d_qual, d_off = (torch.from_numpy(x).cuda() for x in (buf, qual, off))
    sets = [(('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))]
    adapters = fastq._middle_adapters(fastq._norm_sets(sets))
    sides = (wl.pack_adapters([yt]) + ([],), wl.pack_adapters([yb]) + ([],))
    mid = wl.pack_adapters([a[1] for a in adapters])
    h_seq = torch.empty(len(buf), dtype=torch.uint8, pin_memory=True)
    h_qual = torch.empty(len(buf), dtype=torch.uint8, pin_memory=True)
    opts = dict(min_split_read_size=1000)

    def path_a():
        t0 = time.perf_counter()
        st, et, _, _, n_hits, h = W.adapter_trim_reads_device(d_seq.data_ptr(), d_off.data_ptr(), n_reads, len(buf), -1, sides[0],
                                                              sides[1], mid, DEFAULT, 150, 2, 75.0, 4, 85.0,
                                                              stream_ptr=torch.cuda.current_stream().cuda_stream)
        t1 = time.perf_counter()
        h_seq.copy_(d_seq, non_blocking=True)
        h_qual.copy_(d_qual, non_blocking=True)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        batch = fastq.FastqBatch(names, name_off, h_seq.numpy(), off, h_qual.numpy(), off, rna)
        hits = fastq._hits_dict(n_hits, h)
        middle = fastq.middle_trim_ranges(hits, adapters, {'SQK-NSK007_Y_Top'}, {'SQK-NSK007_Y_Bottom'}, 10, 100)
        out = fastq.emit(batch, st, et, middle, 'fastq', opts['min_split_read_size'], as_array=True)
        t3 = time.perf_counter()
        return out, len(h), {'call': t1 - t0, 'copy_home': t2 - t1, 'host_cut': t3 - t2, 'total': t3 - t0}

    def path_b():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = device_reads.trim_reads(d_seq, d_off, sets, DEFAULT, d_qual, **opts)
        torch.cuda.synchronize()
        return r, {'total': time.perf_counter() - t0}

    # warm-up (module load, engine buffers, pinned staging), then the identity check at the timed size
    out_a, n_hits_total, _ = path_a()
    r, _ = path_b()
    parts = tuple(x.cpu().numpy() for x in r[:5])
    same = bytes(out_a) == fastq.emit_parts(names, name_off, rna, parts, 'fastq')
    n_parts, n_out = len(parts[3]), len(parts[0])
    times = {'a': [], 'b': []}
    for _ in range(repeats):
        times['a'].append(path_a()[2])
        times['b'].append(path_b()[1])

    # same-size device-to-device copy (bases + qualities of the output), the practical ceiling of the gather
    src = torch.empty(2 * n_out, dtype=torch.uint8, device='cuda')
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

    # kernel times of one call of path (b), in a run of its own
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
    gather_ms = sum(v for k, v in kern.items() if 'split_gather_kernel' in k)
    stage_ms = sum(v for k, v in kern.items() if 'split_' in k)
    total_kernel_ms = sum(v for k, v in kern.items() if 'Memcpy' not in k and 'Memset' not in k)
    moved = 2 * 2 * n_out                                   # bases + qualities, read once and written once

    hits_bytes = n_hits_total * W.HIT_INTS * 4
    decisions = n_reads * 4 * 3 + hits_bytes                # two trims and n_hits per read, the hit records
    pcie = {'a': decisions + 2 * len(buf),                  # + every base and quality copied home
            'b': decisions + n_hits_total * 16 + 16}        # + the CSR of hit ranges going up (<= 16 B per hit), two totals
    med = lambda xs: float(np.median(xs))                   # noqa: E731
    res = {
        'gpu': gpu_conditions(), 'torch_device': torch.cuda.get_device_name(0),
        'reads': n_reads, 'bases': int(len(buf)), 'records': n_parts, 'out_bases': n_out, 'hits': n_hits_total,
        'identical_output': bool(same), 'repeats': repeats,
        'a_seconds': {k: med([t[k] for t in times['a']]) for k in times['a'][0]},
        'a_total_all': [t['total'] for t in times['a']],
        'b_seconds': med([t['total'] for t in times['b']]), 'b_total_all': [t['total'] for t in times['b']],
        'profile_ms': {'output_stage_split_kernels': stage_ms, 'gather': gather_ms, 'all_kernels': total_kernel_ms},
        'output_stage_share_of_kernel_time': stage_ms / total_kernel_ms if total_kernel_ms else None,
        'gather_TBps': moved / (gather_ms * 1e-3) / 1e12 if gather_ms else None,
        'memcpy_d2d_TBps': moved / (memcpy_ms * 1e-3) / 1e12, 'datasheet_TBps': HBM_TBPS,
        'pcie_bytes': pcie,
    }
    print(json.dumps(res, indent=1))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, 'w') as f:
            json.dump(res, f, indent=1)
    return res


if __name__ == '__main__':
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--reads', type=int, nargs='+', default=[200000])
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default='')
    a = ap.parse_args()
    for n in a.reads:
        run(n, a.repeats, a.out.replace('.json', '_%d.json' % n) if a.out else '')
