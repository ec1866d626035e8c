"""CPU tier, on the host-simulated engine (tests/sim): batches that only the single-pass trace kernel reads (no generic class,
every read <= direct_max) are staged from the caller's ASCII bytes, which trace_kernel encodes through a shared-memory code
table as it stages them, so the call launches no encode pass.  Checked here: the records still equal the oracle's for reads
with mixed case, U, N and bytes outside ACGTUN, through the device-resident and the host-buffer API, and the encode launches
are gone from those calls.  Calls that need the codes (reads longer than direct_max) keep their encode pass."""
import os
import random
import sys

import numpy as np
import pytest

from helpers import ROOT, oracle_batch

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))


@pytest.fixture(scope='module')
def W():
    import sim_engine
    return sim_engine.load()


def _odd_windows(n, w, seed):
    """n reads of length w built from the two NSK007 adapters with their bases in random case, T -> U, N and other bytes"""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    rng = random.Random(seed)
    odd = 'NnUuRYKMSWBDHVryx-.*#@\x01\xff '
    reads = []
    for i in range(n):
        core = (yt if i % 2 else yb) + ''.join(rng.choice('ACGT') for _ in range(w))
        start = rng.randrange(0, len(core) - w + 1)
        r = []
        for ch in core[start:start + w]:
            x = rng.random()
            if x < 0.25:
                ch = ch.lower()
            elif x < 0.30 and ch == 'T':
                ch = rng.choice('Uu')
            elif x < 0.36:
                ch = rng.choice(odd)
            r.append(ch)
        reads.append(bytes(ord(c) & 0xFF for c in r))
    lens = [len(r) for r in reads]
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    return np.frombuffer(b''.join(reads), dtype=np.uint8).copy(), off


def _launches(W, fn):
    n0 = W.kernel_launches()
    fn()
    return W.kernel_launches() - n0


def test_device_resident_ascii_staging_matches_oracle_without_encode(W):
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    buf, off = _odd_windows(300, 150, seed=11)
    ragged_buf, ragged_off = _odd_windows(40, 97, seed=12)
    ragged_off = np.concatenate([ragged_off[:1], ragged_off[1:] - np.arange(1, 41) % 5])    # lengths 92..97
    for buf, off in ((buf, off), (ragged_buf[:ragged_off[-1]].copy(), ragged_off)):
        for ads in ([yt], [yt, yb]):
            abuf, aoff = wl.pack_adapters(ads)
            exp = oracle_batch(buf, off, abuf, aoff, wl.DEFAULT_SCORING)
            out = np.zeros(((len(off) - 1) * len(ads), 9), dtype=np.int32)

            def call(max_len):
                out[:] = 0
                W.adapter_alignment_batch_device(buf.ctypes.data, off.ctypes.data, len(off) - 1, len(buf), max_len, abuf, aoff,
                                                 wl.DEFAULT_SCORING, out.ctypes.data, 0)
                W.synchronize()

            max_len = int(np.diff(off).max())
            call(max_len)                                # plans the adapters (their own encode launch) once
            assert np.array_equal(out, exp)
            # one class, one single-pass trace launch and nothing else; an unknown max_len adds the max_len_kernel
            assert _launches(W, lambda: call(max_len)) == 1
            assert np.array_equal(out, exp)
            assert _launches(W, lambda: call(-1)) == 2
            assert np.array_equal(out, exp)


def test_host_batches_ascii_staging_matches_oracle_without_encode(W):
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    buf, off = _odd_windows(500, 150, seed=13)
    abuf, aoff = wl.pack_adapters([yt, yb])
    exp = oracle_batch(buf, off, abuf, aoff, wl.DEFAULT_SCORING)
    assert np.array_equal(W.adapter_alignment_batch(buf, off, abuf, aoff, wl.DEFAULT_SCORING), exp)
    got = []
    # one chunk of equally long reads: the offsets kernel and the trace launch, no encode
    assert _launches(W, lambda: got.append(W.adapter_alignment_batch(buf, off, abuf, aoff, wl.DEFAULT_SCORING))) == 2
    assert np.array_equal(got[-1], exp)
    # reads longer than direct_max take the two-pass path, which reads codes: the encode pass stays
    lbuf, loff = wl.synth_reads(4, yt, yb, seed=14, chimera_p=0.5, max_len=2000)
    lbuf = lbuf.copy()
    lbuf[::7] = np.frombuffer(b'u', dtype=np.uint8)[0]
    lbuf[3::11] = np.frombuffer(b'n', dtype=np.uint8)[0]
    exp = oracle_batch(lbuf, loff, abuf, aoff, wl.DEFAULT_SCORING)
    assert np.array_equal(W.adapter_alignment_batch(lbuf, loff, abuf, aoff, wl.DEFAULT_SCORING), exp)
