#!/usr/bin/env python3
"""Where the end-trim trace launches spend their time: the same launches timed with builds that leave parts of trace_kernel out.

    python tools/trace_phase_cost.py [--reads 1000000] [--runs 3] [--steps 10] [--warmup 3] [--build-only] [--json FILE]

Every variant is the engine compiled into its own copy of the package (under build/trace_phase_cost/, git-ignored) with
compile-time experiment macros passed through PB200_NVCC_FLAGS:

    default     the shipped kernel
    no_tb       -DPB_EXPERIMENT_SKIP_TRACEBACK: forward pass, scout and stores of the trace only (no records)
    all_hot     -DPB_EXPERIMENT_ALL_HOT: every 4-step chunk, ramp-up and final columns included, runs the unrolled hot chunk
                (clamped column index, no final-column scout); its records are wrong, it is for timing only
    all_hot_no_tb  both

The experiment builds' records are never compared with anything.  Each run is a fresh process that aligns the bench.py
end-trim workload (1 M reads x {150x28 Y_Top, 150x22 Y_Bottom}, seed 20260923) with adapterAlignmentBatchDevice and reads
the CUDA-event time of the trace launches (pb200 timing, timing_read_kinds); the variants are alternated run by run.  The card
name, power limit and SM clock are printed next to the numbers.  --build-only compiles the variants and exits (no GPU needed);
a later run reuses a build made from the same sources and flags.
"""
import argparse
import hashlib
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD_ROOT = os.path.join(ROOT, 'build', 'trace_phase_cost')
VARIANTS = {
    'default': '',
    'no_tb': '-DPB_EXPERIMENT_SKIP_TRACEBACK',
    'all_hot': '-DPB_EXPERIMENT_ALL_HOT',
    'all_hot_no_tb': '-DPB_EXPERIMENT_ALL_HOT -DPB_EXPERIMENT_SKIP_TRACEBACK',
}


def build_variant(name, flags):
    """Copy the package into BUILD_ROOT/<name> and compile its engine with `flags`; returns the directory to put on sys.path."""
    top = os.path.join(BUILD_ROOT, name)
    pkg = os.path.join(top, 'porechop_b200')
    srcs = [os.path.join(ROOT, 'porechop_b200', 'csrc', f) for f in ('engine.cu', 'kernels.cuh', 'dp_core.cuh', 'hostpack.cpp')]
    srcs.append(os.path.join(ROOT, 'include', 'porechop_b200.h'))
    so = os.path.join(pkg, 'cpp_functions.so')
    stamp = os.path.join(top, 'stamp')
    h = hashlib.sha256(flags.encode())
    for s in srcs:
        h.update(open(s, 'rb').read())
    key = h.hexdigest()         # a build is reused only for the same sources and flags (copies of the tree keep no mtimes)
    if os.path.exists(so) and os.path.exists(stamp) and open(stamp).read() == key:
        return top
    shutil.rmtree(top, ignore_errors=True)
    shutil.copytree(os.path.join(ROOT, 'porechop_b200'), pkg,
                    ignore=shutil.ignore_patterns('*.so', '*.o', '__pycache__'))
    shutil.copytree(os.path.join(ROOT, 'include'), os.path.join(top, 'include'))
    env = dict(os.environ, PB200_NVCC_FLAGS=flags)
    subprocess.check_call([sys.executable, '-c', 'from porechop_b200 import build; build.build(force=True)'], cwd=top, env=env)
    with open(stamp, 'w') as f:
        f.write(key)
    return top


def child(args):
    """One timed run of the variant whose package is first on sys.path: prints {'trace_ms_per_step': ...}."""
    import numpy as np
    import torch
    from porechop_b200 import cpp_function_wrappers as W
    from porechop_b200 import workloads as wl
    z = np.load(args.child)
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    batches = []
    for name in ('start', 'end'):
        buf, off = z[name + '_buf'], z[name + '_off']
        abuf, aoff = wl.pack_adapters([str(z[name + '_adapter'])])
        db, do = torch.from_numpy(buf).cuda(), torch.from_numpy(off).cuda()
        dout = torch.empty((len(off) - 1, 9), dtype=torch.int32, device='cuda')
        batches.append((db, do, abuf, aoff, dout, int(np.max(np.diff(off)))))
    torch.cuda.synchronize()

    def step():
        for db, do, abuf, aoff, dout, max_len in batches:
            W.adapter_alignment_batch_device(db.data_ptr(), do.data_ptr(), do.numel() - 1, db.numel(), max_len, abuf, aoff,
                                             wl.DEFAULT_SCORING, dout.data_ptr(), stream.cuda_stream)
    for _ in range(max(args.warmup, 1)):
        step()
    W.synchronize()
    W.timing_enable(True)
    W.timing_read_kinds(reset=True)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(args.steps):
        step()
    ev1.record(stream)
    W.synchronize()
    torch.cuda.synchronize()
    kinds = W.timing_read_kinds(reset=True)
    W.timing_enable(False)
    tk = kinds.get('trace_kernel', {'ms': 0.0, 'n': 0})
    print(json.dumps({'trace_ms_per_step': tk['ms'] / args.steps, 'trace_launches_per_step': tk['n'] / args.steps,
                      'step_ms': ev0.elapsed_time(ev1) / args.steps}))


def gpu_info():
    q = 'name,power.limit,clocks.max.sm,clocks.sm'
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader', '-i', '0'], text=True, timeout=30)
        return dict(zip(q.split(','), [x.strip() for x in out.strip().split(',')]))
    except Exception as e:       # no nvidia-smi: the numbers are printed without it
        return {'error': str(e)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--reads', type=int, default=1000000)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--variants', default=','.join(VARIANTS))
    ap.add_argument('--build-only', action='store_true')
    ap.add_argument('--json', default=None, help='also write the results here')
    ap.add_argument('--child', default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    names = [v for v in args.variants.split(',') if v]
    tops = {v: build_variant(v, VARIANTS[v]) for v in names}
    if args.build_only:
        print('built: ' + ', '.join(names))
        return
    sys.path.insert(0, ROOT)
    import numpy as np
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    _, sw, ew = wl.synth_end_windows(args.reads, yt, yb, seed=wl.SEED)
    tmp = tempfile.mkdtemp(prefix='trace_phase_cost_')
    data = os.path.join(tmp, 'endtrim.npz')
    sbuf, soff = wl.windows_to_batch(sw)
    ebuf, eoff = wl.windows_to_batch(ew)
    np.savez(data, start_buf=sbuf, start_off=soff, end_buf=ebuf, end_off=eoff, start_adapter=yt, end_adapter=yb)
    info = gpu_info()
    res = {v: [] for v in names}
    try:
        for run in range(args.runs):
            for v in names:
                env = dict(os.environ, PYTHONPATH=tops[v])
                out = subprocess.check_output([sys.executable, os.path.abspath(__file__), '--child', data, '--steps', str(args.steps),
                                               '--warmup', str(args.warmup)], env=env, cwd=tmp, text=True)
                r = json.loads(out.strip().splitlines()[-1])
                res[v].append(r)
                print('run %d %-14s trace %.4f ms/step (%d launches), step %.4f ms' % (
                    run, v, r['trace_ms_per_step'], r['trace_launches_per_step'], r['step_ms']), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    info_after = gpu_info()
    print('GPU: %s, power limit %s, max SM clock %s, SM clock %s (before) / %s (after)' % (
        info.get('name'), info.get('power.limit'), info.get('clocks.max.sm'), info.get('clocks.sm'), info_after.get('clocks.sm')))
    summary = {}
    for v in names:
        t = [r['trace_ms_per_step'] for r in res[v]]
        summary[v] = {'trace_ms_per_step': t, 'median': statistics.median(t), 'min': min(t), 'max': max(t)}
        print('%-14s trace ms/step: median %.4f  range %.4f .. %.4f' % (v, summary[v]['median'], min(t), max(t)))
    if 'default' in summary:
        base = summary['default']['median']
        for v in names:
            if v != 'default':
                d = base - summary[v]['median']
                print('default - %-14s %+.4f ms/step (%+.1f %% of the default trace launches)' % (v, d, 100.0 * d / base))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump({'gpu': info, 'gpu_after': info_after, 'reads': args.reads, 'steps': args.steps, 'runs': res, 'summary': summary},
                  open(args.json, 'w'), indent=1)


if __name__ == '__main__':
    main()
