#!/usr/bin/env python3
"""Time the flat FASTQ pipeline (porechop_b200/fastq.py) end to end on one GPU: synthetic FASTQ bytes -> parse -> end
trim (Phase B) -> middle scan (Phase C) -> emit, with the per-stage seconds `trim_fastq` reports.  Not a bench.py
metric (bench.py measures the alignment path itself); this is the tool for finding what the CLI-level run is bound by.

    python tools/flat_pipeline_bench.py --reads 200000 --repeat 3
    python tools/flat_pipeline_bench.py --reads 200000 --middle both    # Phase C: host rounds vs adapterMiddleScan
    python tools/flat_pipeline_bench.py --reads 200000 --search both    # Phase A over every read: host vs adapterSetSearch
    python tools/flat_pipeline_bench.py --reads 200000 --trim both      # Phase B + C: two device calls vs adapterTrimReads

--middle host|device|both times Phase C with the host masking rounds (fastq.find_middle_hits' default) and / or the device
scan (PB200_DEVICE_MIDDLE), alternating the two over the same FASTQ; it reports per path the `middle` seconds of trim_fastq,
rounds, hit reads, hits and the bytes Phase C copies in each direction (counted from the shapes of the engine calls), the
card and its power limit, and asserts that both paths write identical bytes.

--search host|device|both times Phase A over every read (check_reads = number of reads, the 236 sequences of the 119 table
sets, what PB200_CHECK_ALL_READS=1 does) with the record path (fastq.search_adapter_sets' default) and / or the device
reduction (PB200_DEVICE_SEARCH), alternating the two over the same FASTQ; it reports per path the seconds of
search_adapter_sets and the bytes it copies in each direction (counted from the shapes of the engine calls), the card and its
power limit, and asserts that both paths return identical scores.

--trim separate|fused|both times Phase B + Phase C with both device switches on (PB200_DEVICE_DECISIONS and
PB200_DEVICE_MIDDLE): adapterEndDecisions over host-cut windows + adapterMiddleScan over host-gathered trimmed reads
('separate') and / or one adapterTrimReads call ('fused'), alternating the two over the same FASTQ; it reports per path the
`end_trim + middle` seconds of trim_fastq (best run and every run), the engine calls and the bytes they copy in each
direction (counted from the shapes of the calls), the card and its power limit, and asserts that both paths write identical
bytes.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def synthetic_fastq(n_reads, seed, mean_len=8000):
    """FASTQ bytes of the bench.py 'middle' read model (SURVEY 8d: log-normal lengths, adapters at the ends, 5 % chimeras)."""
    import numpy as np
    from porechop_b200 import hostio, workloads as wl
    yt, yb = wl.nsk007()
    buf, off = wl.synth_reads(n_reads, yt, yb, seed=seed, chimera_p=0.05)
    n = len(off) - 1
    names = ['@read_%d ch=%d\n' % (i, i % 512) for i in range(n)]
    nbuf = np.frombuffer(''.join(names).encode(), dtype=np.uint8)
    noff = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(x) for x in names], out=noff[1:])
    lens = np.diff(off)
    rec = np.diff(noff) + lens + 3 + lens + 1                # name line, bases, '\n+\n', qualities, '\n'
    roff = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(rec, out=roff[1:])
    out = np.full(int(roff[-1]), ord('5'), dtype=np.uint8)   # qualities are constant '5' (SURVEY 8d)
    for i in range(n):                                       # generator only, not timed
        p = roff[i]
        out[p:p + len(names[i])] = nbuf[noff[i]:noff[i + 1]]
        p += len(names[i])
        out[p:p + lens[i]] = buf[off[i]:off[i + 1]]
        out[p + lens[i]:p + lens[i] + 3] = np.frombuffer(b'\n+\n', dtype=np.uint8)
        out[roff[i + 1] - 1] = 10
    return out.tobytes(), (yt, yb), hostio.LIB is not None


def run(n_reads, repeat, seed=20260923):
    from porechop_b200 import fastq, workloads as wl
    data, (yt, yb), native = synthetic_fastq(n_reads, seed)
    sets = [(('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))]
    best = None
    for _ in range(repeat):
        t0 = time.perf_counter()
        out, info = fastq.trim_fastq(data, sets, wl.DEFAULT_SCORING, as_array=True)
        total = time.perf_counter() - t0
        if best is None or total < best['seconds_total']:
            best = {'seconds_total': total, 'seconds': info['seconds'], 'out_bytes': int(len(out)),
                    'split_reads': len(info['middle'])}
    best.update({'reads': n_reads, 'in_bytes': len(data), 'reads_per_s': n_reads / best['seconds_total'],
                 'in_MB_per_s': len(data) / 1e6 / best['seconds_total'], 'native_hostio': native})
    return best


def card():
    """name and power limit of the GPU the numbers were measured on (read in the same run)"""
    import subprocess
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=60)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def _phase_c_counter(fastq):
    """wraps the engine calls of find_middle_hits: rounds and bytes each way, from the shapes of what crosses the C-ABI"""
    W = fastq.W
    st = {'rounds': 0, 'h2d_bytes': 0, 'd2h_bytes': 0}
    inside = [False]
    orig_find, orig_batch, orig_scan = fastq.find_middle_hits, W.adapter_alignment_batch, W.adapter_middle_scan

    def find(*a, **k):
        inside[0] = True
        try:
            return orig_find(*a, **k)
        finally:
            inside[0] = False

    def batch(seq_buf, seq_off, ad_buf, ad_off, scoring, pair_seq=None, pair_adapter=None, out=None):
        r = orig_batch(seq_buf, seq_off, ad_buf, ad_off, scoring, pair_seq, pair_adapter, out)
        if inside[0]:
            st['rounds'] += 1
            st['h2d_bytes'] += seq_buf.nbytes + seq_off.nbytes + ad_buf.nbytes + ad_off.nbytes + \
                (pair_seq.nbytes + pair_adapter.nbytes if pair_seq is not None else 0)
            st['d2h_bytes'] += r.nbytes
        return r

    def scan(seq_buf, seq_off, ad_buf, ad_off, scoring, thr):
        n_hits, hits = orig_scan(seq_buf, seq_off, ad_buf, ad_off, scoring, thr)
        rounds = int(n_hits.max()) + 1 if len(n_hits) else 0
        st['rounds'] += rounds
        st['h2d_bytes'] += seq_buf.nbytes + seq_off.nbytes + ad_buf.nbytes + ad_off.nbytes
        st['d2h_bytes'] += rounds * 16 + len(hits) * (4 + hits.shape[1] * 4)   # per round: count, longest read, status
        return n_hits, hits
    return st, (find, batch, scan), (orig_find, orig_batch, orig_scan)


def run_middle(n_reads, repeat, which, seed=20260923):
    import hashlib
    from porechop_b200 import fastq, workloads as wl
    data, (yt, yb), _ = synthetic_fastq(n_reads, seed)
    sets = [(('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))]
    paths = ['host', 'device'] if which == 'both' else [which]
    res, digests = {p: None for p in paths}, {}
    for _ in range(repeat):
        for p in paths:                                       # alternated: the host's other work hits both alike
            st, (find, batch, scan), orig = _phase_c_counter(fastq)
            fastq.find_middle_hits, fastq.W.adapter_alignment_batch, fastq.W.adapter_middle_scan = find, batch, scan
            fastq.DEVICE_MIDDLE = p == 'device'
            try:
                out, info = fastq.trim_fastq(data, sets, wl.DEFAULT_SCORING, as_array=True)
            finally:
                fastq.find_middle_hits, fastq.W.adapter_alignment_batch, fastq.W.adapter_middle_scan = orig
                fastq.DEVICE_MIDDLE = False
            digests.setdefault(p, hashlib.sha256(out).hexdigest())
            assert digests[p] == hashlib.sha256(out).hexdigest()
            m = info['middle']
            cur = {'middle_s': info['seconds']['middle'], 'rounds': st['rounds'], 'hit_reads': len(m),
                   'hits': sum(len(v) for v in m.values()), 'h2d_bytes': st['h2d_bytes'], 'd2h_bytes': st['d2h_bytes']}
            if res[p] is None or cur['middle_s'] < res[p]['middle_s']:
                res[p] = cur
    if len(paths) == 2:
        assert digests['host'] == digests['device'], 'host and device middle scans wrote different output'
    return {'reads': n_reads, 'in_bytes': len(data), 'card': card(), 'repeat': repeat, 'identical_output': len(set(digests.values())) == 1,
            'paths': res}


def _trim_counter(W):
    """wraps the engine calls of Phase B + Phase C with both device switches on: calls and bytes each way, from the shapes of
    what crosses the C-ABI (per masking round: hit count, longest read and status word come back)"""
    st = {'calls': 0, 'h2d_bytes': 0, 'd2h_bytes': 0}
    orig = (W.adapter_end_decisions, W.adapter_middle_scan, W.adapter_trim_reads)

    def hit_bytes(n_hits, hits):
        rounds = int(n_hits.max()) + 1 if len(n_hits) else 0
        return rounds * 16 + len(hits) * (4 + hits.shape[1] * 4)

    def dec(batches, scoring, *a, **k):
        outs = orig[0](batches, scoring, *a, **k)
        st['calls'] += 1
        for b, (trim, scores, _) in zip(batches, outs):
            st['h2d_bytes'] += sum(x.nbytes for x in b[:4]) + 4 * len(b[5] or ())
            st['d2h_bytes'] += trim.nbytes + scores.nbytes
        return outs

    def scan(seq_buf, seq_off, ad_buf, ad_off, scoring, thr):
        n_hits, hits = orig[1](seq_buf, seq_off, ad_buf, ad_off, scoring, thr)
        st['calls'] += 1
        st['h2d_bytes'] += seq_buf.nbytes + seq_off.nbytes + ad_buf.nbytes + ad_off.nbytes
        st['d2h_bytes'] += hit_bytes(n_hits, hits)
        return n_hits, hits

    def trim(seq_buf, seq_off, start, end, middle, *a, **k):
        r = orig[2](seq_buf, seq_off, start, end, middle, *a, **k)
        st['calls'] += 1
        st['h2d_bytes'] += seq_buf.nbytes + seq_off.nbytes + sum(x[0].nbytes + x[1].nbytes + 4 * len(x[2]) for x in (start, end)) + \
            (middle[0].nbytes + middle[1].nbytes if middle is not None else 0)
        st['d2h_bytes'] += r[0].nbytes + r[1].nbytes + r[2].nbytes + r[3].nbytes + hit_bytes(r[4], r[5])
        return r
    return st, (dec, scan, trim), orig


def run_trim(n_reads, repeat, which, seed=20260923):
    """Phase B + Phase C with both device switches on: adapterEndDecisions + adapterMiddleScan ('separate') against one
    adapterTrimReads call ('fused'), alternated over the same FASTQ"""
    import hashlib
    from porechop_b200 import fastq, workloads as wl
    data, (yt, yb), _ = synthetic_fastq(n_reads, seed)
    sets = [(('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))]
    paths = ['separate', 'fused'] if which == 'both' else [which]
    res, digests = {p: None for p in paths}, {}
    W = fastq.W
    fastq.DEVICE_DECISIONS = fastq.DEVICE_MIDDLE = True
    try:
        warm, _, _ = synthetic_fastq(max(n_reads // 50, 1), seed + 1)
        for p in paths:                                       # warm-up: plans, buffers, modules
            fastq.trim_fastq(warm, sets, wl.DEFAULT_SCORING, as_array=True, device_trim=p == 'fused')
        for _ in range(repeat):
            for p in paths:                                   # alternated: the host's other work hits both alike
                st, (dec, scan, trim), orig = _trim_counter(W)
                W.adapter_end_decisions, W.adapter_middle_scan, W.adapter_trim_reads = dec, scan, trim
                try:
                    out, info = fastq.trim_fastq(data, sets, wl.DEFAULT_SCORING, as_array=True, device_trim=p == 'fused')
                finally:
                    W.adapter_end_decisions, W.adapter_middle_scan, W.adapter_trim_reads = orig
                digests.setdefault(p, hashlib.sha256(out).hexdigest())
                assert digests[p] == hashlib.sha256(out).hexdigest()
                s = info['seconds']
                cur = {'end_trim_middle_s': s['end_trim'] + s['middle'], 'end_trim_s': s['end_trim'], 'middle_s': s['middle'],
                       'engine_calls': st['calls'], 'h2d_bytes': st['h2d_bytes'], 'd2h_bytes': st['d2h_bytes'],
                       'split_reads': len(info['middle'])}
                if res[p] is None:
                    res[p] = dict(cur, runs_end_trim_middle_s=[])
                res[p]['runs_end_trim_middle_s'].append(cur['end_trim_middle_s'])
                if cur['end_trim_middle_s'] <= min(res[p]['runs_end_trim_middle_s']):
                    res[p].update(cur)
    finally:
        fastq.DEVICE_DECISIONS = fastq.DEVICE_MIDDLE = False
    if len(paths) == 2:
        assert digests['separate'] == digests['fused'], 'the separate and the fused calls wrote different output'
    return {'reads': n_reads, 'in_bytes': len(data), 'card': card(), 'repeat': repeat,
            'identical_output': len(set(digests.values())) == 1, 'paths': res}


def _phase_a_counter(W):
    """wraps the engine calls of search_adapter_sets: bytes each way, from the shapes of what crosses the C-ABI"""
    st = {'h2d_bytes': 0, 'd2h_bytes': 0}
    orig_batch, orig_search = W.adapter_alignment_batch, W.adapter_set_search

    def batch(seq_buf, seq_off, ad_buf, ad_off, scoring, pair_seq=None, pair_adapter=None, out=None):
        r = orig_batch(seq_buf, seq_off, ad_buf, ad_off, scoring, pair_seq, pair_adapter, out)
        st['h2d_bytes'] += seq_buf.nbytes + seq_off.nbytes + ad_buf.nbytes + ad_off.nbytes
        st['d2h_bytes'] += r.nbytes
        return r

    def search(batches, scoring):
        got = orig_search(batches, scoring)
        for b, g in zip(batches, got):
            st['h2d_bytes'] += sum(x.nbytes for x in b[:4])
            st['d2h_bytes'] += 3 * g.nbytes                   # one u64 key per adapter in each of the engine's 3 stage slices
        return got
    return st, (batch, search), (orig_batch, orig_search)


def run_search(n_reads, repeat, which, seed=20260923):
    import numpy as np
    from porechop_b200 import fastq, workloads as wl
    data, _, _ = synthetic_fastq(n_reads, seed)
    batch = fastq.parse_fastq(data)
    sets = [(d['name'], d['start'] or None, d['end'] or None) for d in wl.load_adapter_sets()['sets']]
    n_seqs = sum(bool(s) + bool(e) for _, s, e in sets)
    paths = ['host', 'device'] if which == 'both' else [which]
    res, scores = {p: None for p in paths}, {}
    W = fastq.W
    fastq.search_adapter_sets(batch, sets, wl.DEFAULT_SCORING, 1000)           # warm-up: plans, buffers, modules
    fastq.search_adapter_sets(batch, sets, wl.DEFAULT_SCORING, 1000, device=True)
    for _ in range(repeat):
        for p in paths:                                       # alternated: the host's other work hits both alike
            st, (b, s), orig = _phase_a_counter(W)
            W.adapter_alignment_batch, W.adapter_set_search = b, s
            try:
                t0 = time.perf_counter()
                got = fastq.search_adapter_sets(batch, sets, wl.DEFAULT_SCORING, len(batch), device=p == 'device')
                sec = time.perf_counter() - t0
            finally:
                W.adapter_alignment_batch, W.adapter_set_search = orig
            scores.setdefault(p, got)
            assert all(np.array_equal(a, b) for a, b in zip(scores[p], got))
            cur = {'phase_a_s': sec, 'h2d_bytes': st['h2d_bytes'], 'd2h_bytes': st['d2h_bytes']}
            if res[p] is None or cur['phase_a_s'] < res[p]['phase_a_s']:
                res[p] = cur
    identical = all(all(np.array_equal(a, b) for a, b in zip(scores[paths[0]], scores[p])) for p in paths)
    if len(paths) == 2:
        assert identical, 'host and device adapter-set searches returned different scores'
    return {'reads': n_reads, 'in_bytes': len(data), 'sequences': n_seqs, 'card': card(), 'repeat': repeat,
            'identical_scores': identical, 'sets_found': int(sum(max(x, y) >= 90.0 for x, y in zip(*scores[paths[0]]))),
            'paths': res}


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--reads', type=int, default=100000)
    ap.add_argument('--repeat', type=int, default=3)
    ap.add_argument('--middle', choices=['host', 'device', 'both'], default=None,
                    help='time Phase C with the host rounds, the device scan, or both alternately')
    ap.add_argument('--search', choices=['host', 'device', 'both'], default=None,
                    help='time Phase A over every read with the record path, the device reduction, or both alternately')
    ap.add_argument('--trim', choices=['separate', 'fused', 'both'], default=None,
                    help='time Phase B + C with the two device calls, the one fused call, or both alternately')
    a = ap.parse_args()
    if a.trim:
        print(json.dumps(run_trim(a.reads, a.repeat, a.trim)))
    elif a.search:
        print(json.dumps(run_search(a.reads, a.repeat, a.search)))
    elif a.middle:
        print(json.dumps(run_middle(a.reads, a.repeat, a.middle)))
    else:
        print(json.dumps(run(a.reads, a.repeat)))
