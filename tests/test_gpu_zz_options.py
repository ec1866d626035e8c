"""GPU tier (pytest -m gpu): engine options and the entry points beyond the plain batch call -- packed upload (h2d_pack),
window bounds (tight_window on / off), query profile of the score pass (profile on / off), global staging (hbuf), the multi
submit, device decisions, error paths.  No option may change a single record.  (Opt-in paths that did not win were
removed.)  The file sorts last on purpose."""
import random

import numpy as np
import pytest

from helpers import oracle_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def W():
    from porechop_b200 import cpp_function_wrappers as w
    assert w.device_count() > 0
    return w


def _with(W, opts, fn):
    defaults = {'hbuf': 'auto', 'h2d_pack': 0, 'tight_window': 1, 'profile': 1, 'direct_max': 160, 'chunk_tasks': 131072, 'pack_threads': 8}
    try:
        for k, v in opts.items():
            W.set_option(k, v)
        return fn()
    finally:
        for k in opts:
            W.set_option(k, defaults[k])


def test_packed_upload_windows_ragged_and_long_reads(W):
    """h2d_pack: Dna5 conversion + 4-bit packing on the host, unpack_kernel on the device -- same records as the oracle
    for end windows (several pipeline chunks), ragged / non-ACGT / empty inputs and long reads (two-pass path)."""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    _, sw, ew = wl.synth_end_windows(30000, yt, yb, seed=77)
    sbuf, soff = wl.windows_to_batch(sw)
    abuf, aoff = wl.pack_adapters([yt, yb])
    exp = oracle_batch(sbuf, soff, abuf, aoff, wl.DEFAULT_SCORING)
    for opts in ({'h2d_pack': 1}, {'h2d_pack': 1, 'chunk_tasks': 9000, 'pack_threads': 3}):
        got = _with(W, opts, lambda: W.adapter_alignment_batch(sbuf, soff, abuf, aoff, wl.DEFAULT_SCORING))
        assert np.array_equal(got, exp), opts
    rng = random.Random(5)
    reads = ['', 'A', 'N' * 21, '-' * 20, 'acgu' * 10, yt, yt[5:], 'GG' + yt + 'GG', 'ACGT' * 301]
    reads += [''.join(rng.choice('ACGTNacgtu-*') for _ in range(rng.randint(1, 401))) for _ in range(300)]
    rbuf, roff = W.pack_sequences(reads)
    got = _with(W, {'h2d_pack': 1}, lambda: W.adapter_alignment_batch(rbuf, roff, abuf, aoff, wl.DEFAULT_SCORING))
    assert np.array_equal(got, oracle_batch(rbuf, roff, abuf, aoff, wl.DEFAULT_SCORING))
    lbuf, loff = wl.synth_reads(40, yt, yb, seed=12, chimera_p=0.4, max_len=15000)
    got = _with(W, {'h2d_pack': 1}, lambda: W.adapter_alignment_batch(lbuf, loff, abuf, aoff, wl.DEFAULT_SCORING))
    assert np.array_equal(got, oracle_batch(lbuf, loff, abuf, aoff, wl.DEFAULT_SCORING))


def test_tight_window_long_reads_and_forced_two_pass_windows(W):
    """tight_window (default) and the per-adapter bound (tight_window=0): second-pass windows sized from the end cell's row
    and score (dp_core.cuh window_cols) or from the adapter length alone.  Long reads
    with 22 / 28 / 111-nt adapters, a masked re-alignment round, cheap-gap schemes, and 150-column windows forced
    through the two-pass path (direct_max = 100) -- identical to the oracle, and to the default windows."""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    full = wl.demux_adapters()[0][-1]
    buf, off = wl.synth_reads(80, yt, yb, seed=41, chimera_p=0.4, max_len=16000)
    abuf, aoff = wl.pack_adapters([yt, yb, full])
    for sc in (wl.DEFAULT_SCORING, (5, -4, -8, -1), (3, -6, -5, -5)):
        exp = oracle_batch(buf, off, abuf, aoff, sc)
        for opts in ({}, {'tight_window': 0}):
            got = _with(W, opts, lambda: W.adapter_alignment_batch(buf, off, abuf, aoff, sc))
            assert np.array_equal(got, exp), (sc, opts)
    masked = buf.copy()
    recs = exp.reshape(80, 3, 9)
    for r in range(80):
        rs, re_ = recs[r, 0, 0], recs[r, 0, 1] + 1
        if rs >= 0:
            masked[off[r] + rs: off[r] + re_] = ord('-')
    got = W.adapter_alignment_batch(masked, off, abuf, aoff, (3, -6, -5, -5))
    assert np.array_equal(got, oracle_batch(masked, off, abuf, aoff, (3, -6, -5, -5)))
    _, sw, ew = wl.synth_end_windows(20000, yt, yb, seed=9)
    for win, ad in ((sw, yt), (ew, yb)):
        sbuf, soff = wl.windows_to_batch(win)
        a1, o1 = wl.pack_adapters([ad])
        exp = oracle_batch(sbuf, soff, a1, o1, wl.DEFAULT_SCORING)
        for opts in ({'direct_max': 100}, {'direct_max': 100, 'tight_window': 0}):
            got = _with(W, opts, lambda: W.adapter_alignment_batch(sbuf, soff, a1, o1, wl.DEFAULT_SCORING))
            assert np.array_equal(got, exp), opts


def test_multi_batch_submit_equals_single_calls(W):
    """adapterAlignmentBatchMulti: several cross-product batches through one ring of streams -- same records as one
    adapterAlignmentBatch call per batch (and the oracle); more distinct adapter lists than the 4-entry plan cache;
    batches of very different sizes; an empty batch in the middle."""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    starts, ends = wl.demux_adapters()
    _, sw, ew = wl.synth_end_windows(150000, yt, yb, seed=3)
    _, sw2, ew2 = wl.synth_end_windows(700, starts[7], ends[7], seed=4)
    lbuf, loff = wl.synth_reads(24, yt, yb, seed=6, chimera_p=0.5, max_len=9000)
    batches = [wl.windows_to_batch(sw) + wl.pack_adapters([yt]),
               wl.windows_to_batch(ew) + wl.pack_adapters([yb]),
               wl.windows_to_batch(sw2) + wl.pack_adapters(starts[:40]),
               (np.zeros(0, dtype=np.uint8), np.zeros(1, dtype=np.int64)) + wl.pack_adapters([yt]),
               wl.windows_to_batch(ew2) + wl.pack_adapters(ends[:33]),
               (lbuf, loff) + wl.pack_adapters([yt, yb]),
               wl.windows_to_batch(sw2) + wl.pack_adapters(starts[40:47])]
    got = W.adapter_alignment_batch_multi(batches, wl.DEFAULT_SCORING)
    assert len(got) == len(batches)
    for b, g in zip(batches, got):
        single = W.adapter_alignment_batch(b[0], b[1], b[2], b[3], wl.DEFAULT_SCORING)
        assert np.array_equal(g, single)
    for k in (1, 2, 4, 5, 6):
        b = batches[k]
        assert np.array_equal(got[k], oracle_batch(b[0], b[1], b[2], b[3], wl.DEFAULT_SCORING)), k
    # all options together
    got2 = _with(W, {'h2d_pack': 1, 'tight_window': 0}, lambda: W.adapter_alignment_batch_multi(batches, wl.DEFAULT_SCORING))
    for a, b in zip(got, got2):
        assert np.array_equal(a, b)


def test_end_decisions_on_device_equal_host_rule(W):
    """adapterEndDecisions (decide_kernel): per-read trim amounts and barcode score pairs computed on the device equal
    libhostio's pbioEndTrim / pbioFullScores applied to the records of the ordinary call -- start and end rule, empty and
    short windows, several chunks, several thresholds; optional record copy-back identical too."""
    from porechop_b200 import hostio, workloads as wl
    from porechop_b200.align import _percent_exact
    starts, ends = wl.demux_adapters()
    ads_s = [starts[0], starts[3], starts[100], starts[150], 'ACGT', starts[-1]]
    ads_e = [ends[0], ends[100], ends[-1]]
    _, sw, ew = wl.synth_end_windows(60000, starts[100], ends[100], seed=8)
    rng = np.random.default_rng(4)

    def ragged(win):
        buf, off = wl.windows_to_batch(win)
        lens = np.diff(off).copy()
        lens[::37] = 0
        lens[5::41] = rng.integers(1, 60, len(lens[5::41]))
        off2 = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        keep = np.repeat(np.arange(len(lens)) * 150, lens) + (np.arange(int(lens.sum())) - np.repeat(off2[:-1], lens))
        return np.ascontiguousarray(buf[keep]), off2
    (sb, so), (eb, eo) = ragged(sw), ragged(ew)
    sa, sao = wl.pack_adapters(ads_s)
    ea, eao = wl.pack_adapters(ads_e)
    srec = W.adapter_alignment_batch(sb, so, sa, sao, wl.DEFAULT_SCORING).reshape(-1, len(ads_s), 9)
    erec = W.adapter_alignment_batch(eb, eo, ea, eao, wl.DEFAULT_SCORING).reshape(-1, len(ads_e), 9)
    scols, ecols = [2, 0, 5, 2], [1]
    for end_size, extra, thr, min_trim, opts in ((150, 2, 75.0, 4, {}), (150, 0, 90.0, 1, {'chunk_tasks': 50000}),
                                                 (150, 5, 50.0, 10, {'h2d_pack': 1}), (150, 2, 0.0, 4, {})):
        outs = _with(W, opts, lambda: W.adapter_end_decisions(
            [(sb, so, sa, sao, True, scols), (eb, eo, ea, eao, False, ecols)], wl.DEFAULT_SCORING, end_size, extra, thr,
            min_trim, want_records=True))
        for (trim, pairs, rec), full_rec, is_start, cols in ((outs[0], srec, True, scols), (outs[1], erec, False, ecols)):
            assert np.array_equal(rec.reshape(full_rec.shape), full_rec)
            assert np.array_equal(trim.astype(np.int64), hostio.end_trim(full_rec, is_start, end_size, extra, thr, min_trim))
            got = _percent_exact(pairs[:, :, 0], pairs[:, :, 1])
            assert np.array_equal(got, hostio.full_scores(full_rec, cols), equal_nan=True)
    # barcode ranking on the device (top2): best / second-best score column = the first two entries of determine_barcode's
    # stable descending sort, for 0, 1, 2 and many columns (ties are frequent: failed alignments all score 0.0)
    from porechop_b200.fastq import Top2Scores, top2_from_scores
    for scols, ecols, opts in (([2, 0, 5, 1, 3], [1], {}), ([4, 3, 2, 1, 0, 5], [0, 2, 1], {'chunk_tasks': 50000}), ([3], [], {})):
        outs = _with(W, opts, lambda: W.adapter_end_decisions(
            [(sb, so, sa, sao, True, scols), (eb, eo, ea, eao, False, ecols)], wl.DEFAULT_SCORING, 150, 2, 75.0, 4,
            want_top2=True))
        for (trim, top2, _), full_rec, is_start, cols in ((outs[0], srec, True, scols), (outs[1], erec, False, ecols)):
            assert np.array_equal(trim.astype(np.int64), hostio.end_trim(full_rec, is_start, 150, 2, 75.0, 4))
            exp = top2_from_scores(hostio.full_scores(full_rec, cols) if cols else np.zeros((len(full_rec), 0)))
            got = Top2Scores([str(c) for c in cols], top2).ranked()
            for g, e in zip(got, exp):
                assert np.array_equal(g, e)


def test_flat_pipeline_with_device_decisions_matches_reference_cli(W, monkeypatch):
    """trim_fastq / demux_fastq goldens (reference CLI output files) with the end-trim decisions taken on the device."""
    from porechop_b200 import fastq
    import test_fastq_emit as T
    monkeypatch.setattr(fastq, 'DEVICE_DECISIONS', True)
    for case in T.CASES:
        T._run(case)
    for case in T.BARCODE_CASES:
        T._run_demux(case)


def test_bad_sequence_offsets_fail_cleanly_mid_pipeline(W):
    """Cross mode checks the sequence offsets chunk by chunk while the pipeline runs: a non-monotone offset in a late
    chunk returns PB200_ERR_ARG after the earlier chunks were submitted, the streams are drained, and the next call works;
    a decision batch with a window longer than end_size is refused the same way."""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    _, sw, _ = wl.synth_end_windows(300000, yt, yb, seed=5)
    sbuf, soff = wl.windows_to_batch(sw)
    abuf, aoff = wl.pack_adapters([yt])
    bad = soff.copy()
    bad[290001] = bad[290000] - 5
    with pytest.raises(W.EngineError) as e:
        W.adapter_alignment_batch(sbuf, bad, abuf, aoff, wl.DEFAULT_SCORING)
    assert 'error 102' in str(e.value) and 'not monotone' in str(e.value)
    good = W.adapter_alignment_batch(sbuf[:150 * 2000], soff[:2001], abuf, aoff, wl.DEFAULT_SCORING)
    assert np.array_equal(good, oracle_batch(sbuf[:150 * 2000], soff[:2001], abuf, aoff, wl.DEFAULT_SCORING))
    with pytest.raises(W.EngineError) as e:
        W.adapter_end_decisions([(sbuf, soff, abuf, aoff, True, [])], wl.DEFAULT_SCORING, 100, 2, 75.0, 4)
    assert 'error 102' in str(e.value)


def test_query_profile_score_pass_equals_oracle(W):
    """profile (default): score_kernel<.., PROF> (substitution operands from a shared-memory query profile) for classes with
    an even number of adapters, the computed-operand kernel for the others in the same call; both window bounds;
    ragged lengths incl. reads shorter than a segment; a masked re-alignment round through the pair list (classic path)."""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    full = wl.demux_adapters()[0][-1]
    sets = [s_ for s_ in wl.load_adapter_sets()['sets'] if s_['name'].endswith('(forward)')][:5]
    bcs = [s_['start'][1] for s_ in sets] + [s_['end'][1] for s_ in sets]
    buf, off = wl.synth_reads(90, yt, yb, seed=23, chimera_p=0.4, max_len=14000)
    rng = random.Random(2)
    short = [''.join(rng.choice('ACGTN') for _ in range(rng.randint(520, 900))) for _ in range(30)] + ['', 'ACGT' * 200]
    sb2, so2 = W.pack_sequences(short)
    buf2 = np.concatenate([buf, sb2]); off2 = np.concatenate([off, so2[1:] + off[-1]])
    for ads in ([yt, yb], [yt, yb, full], bcs, [yt, yb, full, bcs[0]]):
        abuf, aoff = wl.pack_adapters(ads)
        for sc in (wl.DEFAULT_SCORING, (3, -6, -5, -5)):
            exp = oracle_batch(buf2, off2, abuf, aoff, sc)
            for opts in ({}, {'profile': 0}, {'tight_window': 0}):
                got = _with(W, opts, lambda: W.adapter_alignment_batch(buf2, off2, abuf, aoff, sc))
                assert np.array_equal(got, exp), (len(ads), sc, opts)


def test_small_and_odd_classes_ragged_inputs_both_stagings(W):
    """Classes with one adapter (two reads per slot), two adapters (one read per slot), odd classes, an empty adapter, the
    whole demux cross product; ragged / empty / non-ACGT reads; shared-memory and global staging; forced two-pass."""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    rng = random.Random(31)
    reads = ['', 'A', 'N' * 120, '-' * 130, 'acgu' * 40, yt, 'GG' + yt + 'GG', 'ACGT' * 100]
    reads += [''.join(rng.choice('ACGTN') for _ in range(rng.randint(1, 500))) for _ in range(300)]
    rbuf, roff = W.pack_sequences(reads)
    for ads in (['ACGT' * 5], [yt, yb], ['ACGTTGCA' * 5, 'TTGACCA' * 5], ['ACGT' * 16], [yt, ''], ['N' * 22]):
        abuf, aoff = W.pack_sequences(ads, offset_dtype=np.int32)
        for sc in ([3, -6, -5, -2], [3, -6, -5, -5]):
            exp = oracle_batch(rbuf, roff, abuf, aoff, sc)
            for opts in ({}, {'hbuf': 'global'}, {'direct_max': 200}, {'direct_max': 200, 'profile': 0}):
                got = _with(W, opts, lambda: W.adapter_alignment_batch(rbuf, roff, abuf, aoff, sc))
                assert np.array_equal(got, exp), (ads, sc, opts)
    starts, ends = wl.demux_adapters()
    _, sw, ew = wl.synth_end_windows(300, starts[5], ends[5], seed=6)
    for win, ads in ((sw, starts), (ew, ends), (sw, starts[:4]), (sw, starts[:5]), (ew, [yt, yb, starts[-1]])):
        sbuf, soff = wl.windows_to_batch(win)
        abuf, aoff = wl.pack_adapters(ads)
        exp = oracle_batch(sbuf, soff, abuf, aoff, wl.DEFAULT_SCORING)
        for opts in ({}, {'hbuf': 'global'}):
            got = _with(W, opts, lambda: W.adapter_alignment_batch(sbuf, soff, abuf, aoff, wl.DEFAULT_SCORING))
            assert np.array_equal(got, exp), (len(ads), opts)
    lbuf, loff = wl.synth_reads(30, yt, yb, seed=2, chimera_p=0.5, max_len=9000)
    for ads in ([yt, yb, starts[-1]], starts[:5], starts[:6]):
        abuf, aoff = wl.pack_adapters(ads)
        exp = oracle_batch(lbuf, loff, abuf, aoff, wl.DEFAULT_SCORING)
        for opts in ({}, {'profile': 0}):
            got = _with(W, opts, lambda: W.adapter_alignment_batch(lbuf, loff, abuf, aoff, wl.DEFAULT_SCORING))
            assert np.array_equal(got, exp), (len(ads), opts)


def test_global_staging_under_load_every_window_length_mod_4(W):
    """hbuf=global (a slot's packed bases staged in the warp's global scratch behind its trace): the per-warp scratch
    stride must be a whole number of 128-byte lines for every window length -- discard.global.L2 needs aligned
    addresses and must not drop a neighbouring warp's staged bases (round-1 hardware failure at max_n = 150 with the
    stride rounded to 16 bytes only).  >= 30 000 uniform windows so every resident warp loops, window lengths
    150 / 149 / 151 / 153 / 146 (all residues mod 4), one and two adapters."""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    _, sw, ew = wl.synth_end_windows(30011, yt, yb, seed=37)
    full = np.concatenate([sw, ew[:, :10]], axis=1)           # 160 columns to cut from
    for n_cols in (150, 149, 151, 153, 146):
        sbuf, soff = wl.windows_to_batch(np.ascontiguousarray(full[:, :n_cols]))
        for ads in ([yt], [yt, yb]):
            abuf, aoff = wl.pack_adapters(ads)
            exp = oracle_batch(sbuf, soff, abuf, aoff, wl.DEFAULT_SCORING)
            got = _with(W, {'hbuf': 'global'}, lambda: W.adapter_alignment_batch(sbuf, soff, abuf, aoff, wl.DEFAULT_SCORING))
            assert np.array_equal(got, exp), (n_cols, len(ads))
