"""GPU tier (pytest -m gpu): the real kernels under scoring schemes at the edge of the int16 domain, against the oracle --
bit-exact 9-int records.

The CPU tier runs dp_core.cuh on the host, so it never executes the device branches of the packed primitives (DPX max /
add-max / max3, __vadd2, the predicate-accumulating max2acc, the lop3 xnor, __byte_perm unpacking).  These tests run them
in every row-capacity class at its largest length, one less and its smallest length, under 11 scheme shapes with
A = 4000 // (m+3), the largest |score| the class takes at that length (scheme_edges.edge_cases: 528 cases).  Each case goes
in as a cross product and as a pair list, with its reads of <= 160 bases (single trace pass) and with all its reads: per
class 39 single-pass and 27 two-pass cross submissions (the shapes with go = 0 or ge = 0 have no window bound and stay
single-pass over multi-kb reads).  Every call's path is checked against the engine's timed launch kinds: a trace launch
exactly when an int16 class is involved, a score_kernel launch exactly when the two-pass path is expected."""
import random

import numpy as np
import pytest

import scheme_edges as se
from helpers import oracle_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def W():
    from porechop_b200 import cpp_function_wrappers as w
    assert w.device_count() > 0
    w.timing_read_kinds(reset=True)
    w.timing_enable(True)
    try:
        yield w
    finally:
        w.timing_enable(False)
        w.timing_read_kinds(reset=True)


def _same(got, exp, ctx):
    bad = np.flatnonzero((got != exp).any(axis=1)) if got.shape == exp.shape else [0]
    assert len(bad) == 0, '%s: %d of %d records differ; first at row %d: got %s, oracle %s' % (
        ctx, len(bad), len(exp), bad[0], got[bad[0]].tolist(), exp[bad[0]].tolist())


def check(W, rng, reads, ads, sc, ctx, n_short=None, direct_max=se.DIRECT_MAX, path=True):
    """cross and pair-list submissions of `reads` x `ads` (and of the first n_short reads alone) against one oracle run;
    returns the paths the cross submissions took"""
    sbuf, soff = W.pack_sequences(reads)
    abuf, aoff = W.pack_sequences(ads, offset_dtype=np.int32)
    exp = oracle_batch(sbuf, soff, abuf, aoff, sc)
    na, paths = len(ads), set()
    for nr in sorted({n_short or len(reads), len(reads)}):
        sub = (sbuf[:soff[nr]], soff[:nr + 1], abuf, aoff, sc)
        c = '%s, %d reads' % (ctx, nr)
        _same(W.adapter_alignment_batch(*sub), exp[:nr * na], c + ', cross')
        kinds = W.timing_read_kinds(reset=True)
        classes = {}
        for a in ads:
            k = se.route(sc, len(a))
            if k != se.GENERIC:
                classes[k] = max(classes.get(k, 0), len(a))
        two = any(se.two_pass(sc, m, max(len(r) for r in reads[:nr]), direct_max) for m in classes.values())
        traced = any(k.startswith('trace_kernel') for k in kinds)
        assert not path or (traced == bool(classes) and ('score_kernel' in kinds) == two), (c, sorted(kinds), classes)
        paths.add(se.GENERIC if not classes else 'two_pass' if two else 'single_pass')
        ps = np.array([rng.randrange(nr) for _ in range(rng.randint(1, 2 * nr * na))], dtype=np.int32)
        pa = np.array([rng.randrange(na) for _ in ps], dtype=np.int32)
        _same(W.adapter_alignment_batch(*sub, ps, pa), exp[ps.astype(np.int64) * na + pa], c + ', pair list')
        W.timing_read_kinds(reset=True)
    return paths


def _ctx(c):
    return 'class %d m=%d %s %s' % (c['cls'], c['m'], c['shape'], c['scoring'])


def test_every_class_at_its_domain_edge(W):
    rng = random.Random(11)
    seen = {}
    for c in se.edge_cases():
        seen.setdefault(c['cls'], set()).update(check(W, rng, c['short'] + c['long'], c['adapters'], c['scoring'], _ctx(c),
                                                      n_short=len(c['short']) or None))
    assert all(seen[k] == {'single_pass', 'two_pass'} for k in range(16)), seen


def test_routing_boundaries(W):
    """the same inputs on both sides of A*(m+3) = 4000 (int16 class / generic kernel) for every m <= 256 with (m+3) | 4000,
    and of m = 256 (adapters of 256 and 257 alone and mixed in one call)"""
    rng = random.Random(12)
    for m in [d - 3 for d in range(4, 260) if se.LIMIT % d == 0] + [256]:
        A = se.LIMIT // (m + 3)
        ads = [se.rand_seq(rng, m), se.rand_seq(rng, m)]
        longer = [se.rand_seq(rng, 257), se.rand_seq(rng, 257)]
        for shape in ('all_A', 'cheap_gaps', 'affine_open_A', 'free_open'):
            sc, sc_out = dict(se.edge_schemes(A))[shape], dict(se.edge_schemes(A + 1))[shape]
            short, long_ = se.edge_reads(rng, ads, sc, n_random=4)
            runs = [(sc, ads), (sc_out, ads)] if m < 256 else [(sc, ads), (sc, longer), (sc, ads + longer)]
            for s, a in runs:
                assert (se.route(s, len(a[-1])) == se.GENERIC) == (s is sc_out or len(a[-1]) > 256)
                check(W, rng, short + long_, a, s, 'm=%d %s %s %d adapters' % (m, shape, s, len(a)))


def test_options_on_a_subset(W):
    """query profile and window bound switches, global staging of a single pass over long reads, tiny pipeline chunks"""
    hbuf = {0: 'auto', 1: 'smem', 2: 'global'}
    saved = {k: W.get_option(k) for k in ('profile', 'tight_window', 'hbuf', 'direct_max', 'chunk_tasks')}
    rng = random.Random(13)
    subset = se.edge_cases()[::7]
    try:
        for opts in (dict(profile=0, tight_window=1), dict(profile=1, tight_window=0), dict(profile=0, tight_window=0),
                     dict(hbuf='global', direct_max=100000), dict(chunk_tasks=7)):
            for k, v in opts.items():
                W.set_option(k, v)
            for c in subset:                          # tiny chunks see their own longest read: no path check there
                check(W, rng, c['short'] + c['long'], c['adapters'], c['scoring'], '%s %s' % (opts, _ctx(c)),
                      direct_max=opts.get('direct_max', se.DIRECT_MAX), path='chunk_tasks' not in opts)
            for k in opts:
                W.set_option(k, hbuf[saved[k]] if k == 'hbuf' else saved[k])
    finally:
        for k, v in saved.items():
            W.set_option(k, hbuf[v] if k == 'hbuf' else v)


def test_cheap_gaps_wide_windows_on_multi_kb_reads(W):
    """gap scores far cheaper than the match score: W(m) is many times m, and gappy implants put long read-only gap runs on
    the traced paths"""
    rng = random.Random(14)
    for sc in ([12, -3, -1, -1], [10, -20, -15, -7]):
        ads = [se.rand_seq(rng, m) for m in (7, 24, 28, 33, 70, 128)]
        reads = []
        for _ in range(24):
            r = se.rand_seq(rng, rng.randint(2000, 9000))
            for _ in range(rng.randint(0, 3)):
                r = se.implant(rng, r, se.gappy(rng, rng.choice(ads), p_ins=rng.choice([0.2, 0.5, 0.8])))
            reads.append(r)
        assert check(W, rng, reads, ads, sc, str(sc)) == {'two_pass'}


def test_device_resident_entry_point_equals_host_api(W):
    import torch
    for c in se.edge_cases()[3::11]:
        sc, ads = c['scoring'], c['adapters']
        for reads in (c['short'], c['short'] + c['long']):
            if not reads:
                continue
            sbuf, soff = W.pack_sequences(reads)
            abuf, aoff = W.pack_sequences(ads, offset_dtype=np.int32)
            host = W.adapter_alignment_batch(sbuf, soff, abuf, aoff, sc)
            d_seq = torch.from_numpy(np.concatenate([sbuf, np.zeros(1, np.uint8)])).cuda()
            d_off = torch.from_numpy(soff).cuda()
            d_out = torch.full((len(reads) * len(ads) * 9,), -7, dtype=torch.int32, device='cuda')
            torch.cuda.synchronize()
            W.adapter_alignment_batch_device(d_seq.data_ptr(), d_off.data_ptr(), len(reads), len(sbuf), max(map(len, reads)),
                                             abuf, aoff, sc, d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            W.synchronize()
            _same(d_out.cpu().numpy().reshape(-1, 9), host, 'device API ' + _ctx(c))
    W.timing_read_kinds(reset=True)
