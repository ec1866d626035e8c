#!/usr/bin/env python3
"""Traceback path lengths of the end-trim trace launches, counted on the host-simulated engine (tests/sim).

    python tools/trace_path_steps.py [--reads 4000] [--seed 20260923]

Builds the simulated engine with -DPB_EXPERIMENT_PATH_STEPS (a library of its own; the product build never defines it, and
without it the kernel is unchanged) and aligns the bench.py end-trim windows of `--reads` reads (the same generator and seed,
a prefix-sized sample) against Y_Top / Y_Bottom.  Prints, per side, the mean path length in steps of the traced alignments and
the mean over warp slots of the longest path in the warp -- the warp's traceback lasts as long as that one.  The simulator
runs the kernel's own code, so the counts are the device's; no time is measured.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--reads', type=int, default=4000)
    ap.add_argument('--seed', type=int, default=None)
    args = ap.parse_args()
    import sim_engine
    from porechop_b200 import workloads as wl
    W = sim_engine.load(['-DPB_EXPERIMENT_PATH_STEPS'])
    stats = (ctypes.c_ulonglong * 4).in_dll(W.C_LIB, 'pb_path_stats')
    yt, yb = wl.nsk007()
    _, sw, ew = wl.synth_end_windows(args.reads, yt, yb, seed=wl.SEED if args.seed is None else args.seed)
    res = {}
    for side, win, ad in (('start', sw, yt), ('end', ew, yb)):
        for k in range(4):
            stats[k] = 0
        buf, off = wl.windows_to_batch(win)
        abuf, aoff = wl.pack_adapters([ad])
        W.adapter_alignment_batch(buf, off, abuf, aoff, wl.DEFAULT_SCORING)
        steps, paths, wmax, wslots = (int(stats[k]) for k in range(4))
        res[side] = {'adapter_len': len(ad), 'alignments': paths, 'mean_path_steps': steps / max(paths, 1),
                     'mean_warp_max_path_steps': wmax / max(wslots, 1), 'warp_slots': wslots}
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
