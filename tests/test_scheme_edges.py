"""CPU tier: the class x edge-scheme sweep of tests/scheme_edges.py (run on the GPU by tests/test_gpu_schemes.py) through the
kernel core compiled for the host (tests/emu, with its int16 range check) and through the simulated engine (tests/sim) --
records equal to the oracle's, and not one value outside the int16 domain."""
import ctypes
import os
import random
import sys

import numpy as np

import scheme_edges as se
from helpers import ROOT, emu_lib, emu_slot, oracle_batch
from porechop_b200 import cpp_function_wrappers as W

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))


def test_sweep_sits_at_the_edge_and_covers_every_class_and_path():
    paths = {}
    for c in se.edge_cases():
        sc, m = c['scoring'], c['m']
        A = max(abs(x) for x in sc)
        assert se.route(sc, m) == c['cls'] and A * (m + 3) <= 4000 < (A + 1) * (m + 3), c
        for reads in (c['short'], c['short'] + c['long']):
            if reads:
                two = se.two_pass(sc, m, max(map(len, reads)))
                paths.setdefault((c['cls'], c['shape']), set()).add('two_pass' if two else 'single_pass')
    for k in range(16):
        for shape, sc in se.edge_schemes(10):
            assert paths[k, shape] == ({'single_pass', 'two_pass'} if se.window(sc, 1) else {'single_pass'}), (k, shape)


def _emu_run(tasks, G, R, mode, sc, exp, ctx):
    """tasks: (read, adapter, oracle row); two alignments per slot; no int16 range violation"""
    lib = emu_lib()
    lib.emu_range_violations.restype = ctypes.c_long
    v0 = lib.emu_range_violations()
    for j in range(0, len(tasks), 2):
        pair = tasks[j:j + 2]
        st, ra, rb = emu_slot(pair[0][:2], pair[1][:2] if len(pair) > 1 else None, G, R, mode, sc)
        assert st & 1 == 0, (ctx, mode, pair)
        for t, rec in zip(pair, (ra, rb)):
            assert rec == exp[t[2]].tolist(), (ctx, mode, G, R, t[:2])
    assert lib.emu_range_violations() == v0, (ctx, mode, 'int16 range violations')


def test_emu_edge_sweep():
    """single pass (mode 0) over every read at the class geometry; for schemes with a window bound the two-pass forms over the
    long reads: classic (1) and per-alignment (5) window bound, and the query-profile score pass at R = 8 (9, 13)"""
    rng = random.Random(21)
    for c in se.edge_cases():
        sc, ads = c['scoring'], c['adapters']
        reads = c['short'] + c['long']
        sbuf, soff = W.pack_sequences(reads)
        abuf, aoff = W.pack_sequences(ads, offset_dtype=np.int32)
        exp = oracle_batch(sbuf, soff, abuf, aoff, sc)
        na = len(ads)
        tasks = [(r, a, i * na + j) for i, r in enumerate(reads) for j, a in enumerate(ads)]
        rng.shuffle(tasks)
        G, R = 4 << (c['cls'] // 4), 5 + c['cls'] % 4
        ctx = 'class %d m=%d %s %s' % (c['cls'], c['m'], c['shape'], sc)
        _emu_run(tasks, G, R, 0, sc, exp, ctx)
        if se.window(sc, c['m']) is None:
            continue
        for mode in (1, 5):
            _emu_run([t for t in tasks if len(t[0]) > se.DIRECT_MAX], G, R, mode, sc, exp, ctx)
        same_read = [(r, ads[j], i * na + j) for i, r in enumerate(reads) if len(r) > se.DIRECT_MAX for j in (0, 1)]
        for mode in (9, 13):
            _emu_run(same_read, G, 8, mode, sc, exp, ctx)


def test_sim_engine_edge_sweep():
    """the simulated engine (the product's engine.cu and kernels on the host): cross and pair-list submissions of short reads
    and of all reads, every shape in every class at one of the class's three lengths (rotating with the shape)"""
    import sim_engine
    SW = sim_engine.load()
    sim_engine.clear_races()
    rng = random.Random(22)
    shapes = [s for s, _ in se.edge_schemes(10)]
    for c in se.edge_cases(n_random=3, long_reads=1):
        if c['m'] != se.class_lengths(c['cls'])[shapes.index(c['shape']) % 3]:
            continue
        sc, ads, reads = c['scoring'], c['adapters'], c['short'] + c['long']
        sbuf, soff = SW.pack_sequences(reads)
        abuf, aoff = SW.pack_sequences(ads, offset_dtype=np.int32)
        exp = oracle_batch(sbuf, soff, abuf, aoff, sc)
        na = len(ads)
        for nr in {len(c['short']) or len(reads), len(reads)}:
            sub = (sbuf[:soff[nr]], soff[:nr + 1], abuf, aoff, sc)
            assert np.array_equal(SW.adapter_alignment_batch(*sub), exp[:nr * na]), (c['cls'], c['m'], c['shape'], nr)
            ps = np.array([rng.randrange(nr) for _ in range(nr * na)], dtype=np.int32)
            pa = np.array([rng.randrange(na) for _ in ps], dtype=np.int32)
            assert np.array_equal(SW.adapter_alignment_batch(*sub, ps, pa), exp[ps.astype(np.int64) * na + pa]), \
                (c['cls'], c['m'], c['shape'], nr, 'pair list')
    sim_engine.assert_no_races()
