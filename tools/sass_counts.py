#!/usr/bin/env python3
"""profiles/sass_counts.json: SASS instructions per DP cell in the hot loops of the DP kernels (bench.py `roofline_alu`).

    python tools/sass_counts.py profiles/<round>_trace_kernel.ncu-rep profiles/<round>_score_kernel.ncu-rep ...

Input: `ncu --set full --import-source on` reports of bench.py launches.  For every kernel in a
report the SASS page gives, per instruction, how often it was executed.  The hot loop is the set of instructions that share
the most frequent execution count weighted by its size (the unrolled straight-line step loop: every one of its instructions
runs exactly once per iteration, nothing else in the kernel runs that often AND is that large).  With `steps` wavefront steps
per iteration (trace_kernel: PB_TCHUNK = 4; score_kernel: the `#pragma unroll 4` body) and 2*R cells per lane and step:

    instr_per_cell = hot static instructions / (steps * 2 * R)

That is the issue-slot cost of one cell when every lane is busy and nothing but the step loop runs -- the denominator of
roofline_alu.peak_cells_per_s = SMs * 4 schedulers * 32 lanes * clock / instr_per_cell.  The dynamic share of the hot loop
(hot_dynamic_frac) and the whole-kernel dynamic instructions per cell are recorded next to it.
"""
import csv
import io
import json
import os
import re
import subprocess
import sys
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def kernels_of(rep):
    out = subprocess.run(['ncu', '-i', rep, '--page', 'source', '--csv', '--print-source', 'sass'], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    cur, hdr, res = None, None, []
    for r in rows:
        if r and r[0] == 'Kernel Name':
            cur = {'name': r[1], 'rows': []}
            res.append(cur)
        elif r and r[0] == 'Address':
            hdr = r
        elif cur is not None and hdr is not None and len(r) >= 8 and r[0].startswith('0x'):
            cur['rows'].append(dict(zip(hdr, r)))
    return res


def analyse(k):
    m = re.search(r'(trace_kernel|score_kernel)<\(int\)(\d+), \(int\)(\d+)', k['name'])
    if not m:
        return None
    kind, G, R = m.group(1), int(m.group(2)), int(m.group(3))
    ex = [int(r['Instructions Executed']) for r in k['rows']]
    total = sum(ex)
    cnt = Counter(ex)
    # the class with the largest dynamic share
    hot_count, hot_static = max(cnt.items(), key=lambda kv: kv[0] * kv[1])
    steps = 4
    dpx = sum(1 for r in k['rows'] if int(r['Instructions Executed']) == hot_count and
              re.search(r'VIMNMX|VIADDMNMX|VIADD\.16x2|VIMNMX3', r['Source']))
    return {'kernel': '%s<%d,%d>' % (kind, G, R), 'G': G, 'R': R, 'hot_static_instructions': hot_static,
            'hot_dpx_instructions': dpx, 'steps_per_iteration': steps, 'cells_per_lane_step': 2 * R,
            'instr_per_cell': hot_static / (steps * 2.0 * R), 'hot_dynamic_frac': hot_count * hot_static / max(total, 1),
            'warp_instructions_launch': total, 'static_instructions': len(ex)}


def main():
    res = {}
    for rep in sys.argv[1:]:
        for k in kernels_of(rep):
            a = analyse(k)
            if a is None:
                continue
            a['source'] = 'ncu SASS page of ' + os.path.basename(rep) + ' (tools/sass_counts.py)'
            res.setdefault(a['kernel'], a)
    # bench.py looks the dominant kernel up by family name: the row-capacity class of the headline config
    for fam, pick in (('trace_kernel', 'trace_kernel<4,7>'), ('score_kernel', 'score_kernel<4,8>')):
        if pick in res:
            res[fam] = dict(res[pick])
    os.makedirs(os.path.join(ROOT, 'profiles'), exist_ok=True)      # git-ignored: measured output, per GPU
    p = os.path.join(ROOT, 'profiles', 'sass_counts.json')
    json.dump(res, open(p, 'w'), indent=1, sort_keys=True)
    for k, v in sorted(res.items()):
        print('%-22s hot %4d static (%d DPX) / %d steps x %d cells = %.2f instr/cell, hot share of dynamic %.2f' % (
            k, v['hot_static_instructions'], v['hot_dpx_instructions'], v['steps_per_iteration'], v['cells_per_lane_step'],
            v['instr_per_cell'], v['hot_dynamic_frac']))


if __name__ == '__main__':
    main()
