"""CPU tier: host-side logic -- workloads, packing, the native reference harness, sharding + gather (gloo, 2 ranks)."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

from helpers import ROOT, oracle_batch, oracle_string


def test_workload_determinism_and_shapes():
    from porechop_b200 import workloads as W
    yt, yb = W.nsk007()
    assert (len(yt), len(yb)) == (28, 22)
    L1, s1, e1 = W.synth_end_windows(2000, yt, yb)
    L2, s2, e2 = W.synth_end_windows(2000, yt, yb)
    assert np.array_equal(L1, L2) and np.array_equal(s1, s2) and np.array_equal(e1, e2)
    assert s1.shape == (2000, 150) and set(np.unique(s1)) <= set(b'ACGT')
    assert 6000 < L1.mean() < 10000
    starts, ends = W.demux_adapters()
    assert (len(starts), len(ends)) == (227, 129)
    assert sum(map(len, starts)) + sum(map(len, ends)) == 17975     # SURVEY 8(d) config 3
    # implanted adapters are found by the oracle in most start windows
    hits = 0
    for k in range(60):
        p = oracle_string(bytes(s1[k]).decode(), yt).split(',')
        hits += float(p[5]) > 75.0 and int(p[0]) == 0
    assert hits > 25


def test_pack_sequences_roundtrip():
    from porechop_b200.cpp_function_wrappers import pack_sequences
    seqs = ['ACGT', '', 'NNNA', 'acgu-']
    buf, off = pack_sequences(seqs)
    assert [bytes(buf[off[i]:off[i + 1]]).decode() for i in range(4)] == seqs


def test_reference_harness_matches_oracle_batch():
    from porechop_b200 import workloads as W
    yt, yb = W.nsk007()
    _, sw, _ = W.synth_end_windows(64, yt, yb)
    sbuf, soff = W.windows_to_batch(sw)
    abuf, aoff = W.pack_adapters([yt, yb])
    harness = os.path.join(ROOT, 'oracle', '_ref', 'ref_harness')
    lib = os.path.join(ROOT, 'oracle', '_ref', 'cpp_functions.so')
    if not os.path.exists(lib):
        lib = os.path.join(ROOT, 'oracle', 'liboracle.so')
    with tempfile.TemporaryDirectory() as d:
        wl, ans = os.path.join(d, 'w.bin'), os.path.join(d, 'a.txt')
        W.write_harness_file(wl, sbuf, soff, abuf, aoff, W.DEFAULT_SCORING)
        out = subprocess.check_output([harness, lib, wl, '2', ans]).decode()
        info = json.loads(out)
        assert info['pairs'] == 128 and info['cells'] == 64 * 150 * 50
        got = open(ans).read().split('\n')[:-1]
    from porechop_b200.align import record_string
    exp = [record_string(r) for r in oracle_batch(sbuf, soff, abuf, aoff, W.DEFAULT_SCORING)]
    assert got == exp


def test_shard_bounds():
    from porechop_b200.distributed import shard_bounds, shard_bounds_by_bases
    assert list(shard_bounds(10, 4)) == [0, 3, 6, 8, 10]
    off = np.concatenate([[0], np.cumsum([100, 100, 100, 100, 400, 100, 100])])
    b = shard_bounds_by_bases(off, 2)
    assert b[0] == 0 and b[-1] == 7 and 4 <= b[1] <= 5


def _gather_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from porechop_b200.distributed import gather_records, shard_bounds
    n = 11
    b = shard_bounds(n, world)
    full = torch.arange(n * 9, dtype=torch.int32).reshape(n, 9)
    local = full[b[rank]:b[rank + 1]].clone()
    got = gather_records(local, [int(b[r + 1] - b[r]) for r in range(world)], dst=0)
    if rank == 0:
        q.put(bool(torch.equal(got, full)))
    else:
        q.put(got is None)
    dist.destroy_process_group()


def test_gather_records_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_gather_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(res)


def test_bench_parity_gate_against_harness_answers():
    """bench.py's parity gate (SURVEY 8d): harness answer strings vs records rendered by pb200FormatRecord.  Here the
    records come from the oracle (no GPU in this tier); one record is then corrupted to see the gate fire.  Also the CPU
    baseline block (1 thread + thread / process sweep) and the identical `config` dicts of the two arms."""
    import sys
    sys.path.insert(0, ROOT)
    import bench
    from porechop_b200 import workloads as wl
    from porechop_b200 import cpp_function_wrappers as W
    sys_argv, sys.argv = sys.argv, ['bench.py', '--reads', '200']
    try:
        args = bench.parse_args()
    finally:
        sys.argv = sys_argv
    w = bench.make_workload('endtrim', args, 0, 1, True)
    assert w.n == 200 and len(w.batches) == 2 and w.cells == 200 * 7500
    assert w.config('weak') == bench.make_nominal_config('endtrim', args, True)
    files = bench.HarnessFiles(w, [150, 150])
    answers = []
    sec = files.run(2, 1, answers)
    assert len(answers) == 2 and len(answers[0]) == 150 and sec > 0 and files.cells == 150 * 7500
    assert files.run(1, 2) > 0                                   # forked worker processes, no answers
    recs = []
    for name, buf, off, ads in w.batches:
        abuf, aoff = wl.pack_adapters(ads)
        recs.append(oracle_batch(buf, off, abuf, aoff, wl.DEFAULT_SCORING))
    assert bench.parity_gate(recs, answers, W.format_record) == {'checked': 300, 'mismatches': 0}
    recs[1][3, 1] += 1
    assert bench.parity_gate(recs, answers, W.format_record) == {'checked': 300, 'mismatches': 1}
    cb, ans, sizes = bench.cpu_baseline(w, sample_reads=100, sweep=True)
    assert cb['kind'] in ('reference', 'port') and cb['value'] > 0 and cb['one_thread']['value'] > 0 and len(cb['sweep']) >= 2
    assert cb['host']['nproc'] and len(ans) == 2 and sizes == [100, 100]
    # prefix consistency of the generators the reference arm relies on (same first reads for any batch size)
    for name in ('middle', 'sweep'):
        sys.argv = ['bench.py', '--config-reads', 'middle=300', '--sweep-bases', '60000', '--sweep-lengths', '500,2000']
        try:
            a2 = bench.parse_args()
        finally:
            sys.argv = sys_argv
        full = bench.make_workload(name, a2, 0, 1, False)
        part = bench.make_workload(name, a2, 0, 1, False, limit=7)
        for (n1, b1, o1, _), (n2, b2, o2, _) in zip(full.batches, part.batches):
            k = len(o2) - 1
            assert k >= 1 and np.array_equal(o1[:k + 1], o2) and np.array_equal(b1[:o2[-1]], b2[:o2[-1]])
        assert full.config('weak') == bench.make_nominal_config(name, a2, False)


def test_packed_upload_path_host_pack_and_device_unpack_equal_encode():
    """Option h2d_pack: pb200PackNibbles (hostpack.cpp, AVX2 + scalar tail, any thread count) followed by the device's
    unpack arithmetic (dp_core.cuh unpack_nibbles8 / unpack_nibble1, run on the host by tests/emu) gives exactly the
    code bytes of encode_byte -- for every byte value, every length around the SIMD / work-item boundaries, odd lengths."""
    import ctypes
    from helpers import emu_lib
    from porechop_b200 import cpp_function_wrappers as W
    emu = emu_lib()
    emu.emu_unpack.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
    emu.emu_encode.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
    emu.emu_unpack.restype = emu.emu_encode.restype = None
    rng = np.random.default_rng(11)
    every = np.arange(256, dtype=np.uint8)
    cases = [every, every[::-1].copy(), np.zeros(0, dtype=np.uint8)]
    for n in [1, 2, 3, 15, 16, 17, 31, 32, 33, 63, 64, 65, 1000, 65535, 65536, 65537, 3 * 65536 + 5, 1 << 20]:
        kind = rng.integers(0, 3)
        if kind == 0:
            a = rng.integers(0, 256, n).astype(np.uint8)
        else:
            a = np.frombuffer(b'ACGTUacgtuNn-*', dtype=np.uint8)[rng.integers(0, 14, n)]
        cases.append(np.ascontiguousarray(a))
    for a in cases:
        n = len(a)
        exp = np.zeros(n, dtype=np.uint8)
        emu.emu_encode(a.ctypes.data, exp.ctypes.data, n)
        for threads in (1, 3, 0):
            pk = W.pack_nibbles(a, threads)
            assert len(pk) == (n + 1) // 2
            got = np.zeros(n, dtype=np.uint8)
            emu.emu_unpack(pk.ctypes.data, got.ctypes.data, n)
            assert np.array_equal(got, exp), (n, threads)
    if not os.environ.get('PB200_PACK_NO_AVX512'):          # the AVX2 body on machines that would pick the AVX-512 one
        r = subprocess.run([sys.executable, '-m', 'pytest', '-x', '-q', __file__, '-k', 'packed_upload_path'],
                           env=dict(os.environ, PB200_PACK_NO_AVX512='1'), capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stdout[-1500:]


def test_trim_threshold_table_is_the_exact_float_rule():
    """pb200TrimThresholdTable: `c >= cmin[l]` is exactly the reference's `float("%f" % (100.0*c/l)) > end_threshold`
    (alignment.cpp:113-121 + nanopore_read.py:488) for every count and aligned length, also at thresholds that sit on
    printf's rounding boundaries."""
    from porechop_b200 import cpp_function_wrappers as W
    for thr in (75.0, 90.0, 0.0, 100.0, 50.0, 33.333333, 33.3333335, 66.666667, 66.6666665, 99.999999, 14.285714, 85.5):
        L = 420
        cmin = W.trim_threshold_table(thr, L)
        assert cmin[0] == 2 ** 31 - 1
        for l in range(1, L):
            vals = np.array([float('%f' % (100.0 * c / l)) for c in range(l + 1)])
            ok = vals > thr
            first = int(np.argmax(ok)) if ok.any() else l + 1
            assert cmin[l] == first, (thr, l)
            assert np.array_equal(ok, np.arange(l + 1) >= cmin[l])


def test_device_decision_core_equals_host_trim_rule_and_barcode_scores():
    """The decision kernel's per-record core (dp_core.cuh end_trim_candidate / score_pair, run serially by tests/emu) on
    oracle records: trim amounts equal libhostio's pbioEndTrim (and the numpy rule), and the (match, length) pairs give the
    same doubles as pbioFullScores -- start and end rule, empty windows, several thresholds / window sizes."""
    import ctypes
    from helpers import emu_lib
    from porechop_b200 import cpp_function_wrappers as W, hostio, workloads as wl
    from porechop_b200.align import _percent_exact
    emu = emu_lib()
    emu.emu_decide.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_int, ctypes.c_int32, ctypes.c_int32,
                               ctypes.c_int32, ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p,
                               ctypes.c_void_p]
    emu.emu_decide.restype = ctypes.c_int
    starts, ends = wl.demux_adapters()
    ads = [starts[0], starts[3], starts[100], starts[150], ends[100], 'ACGT', starts[-1]]
    _, sw, ew = wl.synth_end_windows(600, starts[100], ends[100], seed=8)
    rng = np.random.default_rng(2)
    for win, is_start in ((sw, 1), (ew, 0)):
        sbuf, soff = wl.windows_to_batch(win)
        # a few empty and short windows (reads shorter than end_size)
        lens = np.diff(soff).copy()
        lens[::37] = 0
        lens[5::41] = rng.integers(1, 60, len(lens[5::41]))
        off2 = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        buf2 = np.concatenate([sbuf[soff[i]:soff[i] + lens[i]] for i in range(len(lens))]) if len(lens) else sbuf[:0]
        abuf, aoff = wl.pack_adapters(ads)
        rec = oracle_batch(buf2, off2, abuf, aoff, wl.DEFAULT_SCORING).reshape(len(lens), len(ads), 9)
        cols = np.array([2, 0, 6, 2], dtype=np.int32)
        for end_size, extra, thr, min_trim in ((150, 2, 75.0, 4), (150, 0, 90.0, 1), (100, 5, 50.0, 10), (150, 2, 0.0, 4)):
            L = 150 + max(len(a) for a in ads) + 2
            cmin = W.trim_threshold_table(thr, L)
            trim = np.zeros(len(lens), dtype=np.int32)
            pairs = np.zeros((len(lens), len(cols)), dtype=np.uint32)
            flat = np.ascontiguousarray(rec.reshape(-1, 9))
            ovf = emu.emu_decide(flat.ctypes.data, len(lens), len(ads), is_start, end_size, extra, min_trim, cmin.ctypes.data, L,
                                 cols.ctypes.data, len(cols), trim.ctypes.data, pairs.ctypes.data)
            assert ovf == 0
            exp = hostio.end_trim(rec, bool(is_start), end_size, extra, thr, min_trim)
            assert np.array_equal(trim.astype(np.int64), exp), (is_start, end_size, thr)
            full = _percent_exact(pairs & 0xFFFF, pairs >> 16)
            assert np.array_equal(full, hostio.full_scores(rec, [int(c) for c in cols]), equal_nan=True)


def test_unpack_device_branch_byte_perm_selectors():
    """dp_core.cuh unpack_nibbles8 has a device branch (two PRMT: __byte_perm(e, o, 0x5140) / (e, o, 0x7362)) and a generic
    branch; the host tests run the generic one.  The selectors are checked here against PRMT's definition (result byte i =
    byte (selector nibble i) of the 8-byte pair {x = bytes 0-3, y = bytes 4-7})."""
    import ctypes
    from helpers import emu_lib
    emu = emu_lib()
    emu.emu_unpack.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
    emu.emu_unpack.restype = None

    def byte_perm(x, y, s):
        xy = (y << 32) | x
        return sum(((xy >> (8 * ((s >> (4 * i)) & 7))) & 0xFF) << (8 * i) for i in range(4))
    rng = np.random.default_rng(5)
    for w in [0, 0xFFFFFFFF, 0x01234567, 0x40302010] + [int(x) for x in rng.integers(0, 2 ** 32, 500)]:
        e, o = ((w & 0x0F0F0F0F) << 4) & 0xFFFFFFFF, w & 0xF0F0F0F0
        packed = np.frombuffer(np.array([w, w], dtype=np.uint32).tobytes(), dtype=np.uint8).copy()
        out = np.zeros(16, dtype=np.uint8)
        emu.emu_unpack(packed.ctypes.data, out.ctypes.data, 16)
        first4, next4 = np.frombuffer(out[:8].tobytes(), dtype=np.uint32)
        assert int(first4) == byte_perm(e, o, 0x5140) and int(next4) == byte_perm(e, o, 0x7362), hex(w)


def test_simulated_engine_results_do_not_depend_on_lane_interleaving():
    """tests/sim resumes the runnable CUDA threads of a block in index order; the device defines no order between two
    collectives.  Two of the simulated-engine tests again with the order reversed and shuffled (separate processes: the
    order is read once): a missing __syncwarp around shared memory would change the records."""
    for order in ('random:5',):
        env = dict(os.environ, PBSIM_ORDER=order)
        r = subprocess.run([sys.executable, '-m', 'pytest', '-x', '-q', os.path.join(ROOT, 'tests', 'test_sim_engine.py'), '-k',
                            'long_reads_two_pass_and_options or multi_submit'], env=env, capture_output=True,
                           text=True, cwd=ROOT)
        assert r.returncode == 0 and '2 passed' in r.stdout, order + '\n' + r.stdout[-2000:]


def test_cpu_quota_is_respected_by_the_cpu_baseline_sizing_and_hostio(monkeypatch, tmp_path):
    """A host may show many more hardware threads than its cgroup CPU quota lets run.  bench.py sizes the CPU baseline and
    hostio its OpenMP team by what the quota allows, not by the visible threads."""
    import builtins
    import importlib
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    bench = importlib.import_module('bench')
    from porechop_b200 import hostio
    real_open = builtins.open

    def fake_open(quota):
        def _open(path, *a, **k):
            if path == '/sys/fs/cgroup/cpu.max':
                p = tmp_path / 'cpu.max'
                p.write_text(quota)
                return real_open(p, *a, **k)
            return real_open(path, *a, **k)
        return _open
    monkeypatch.setattr(os, 'sched_getaffinity', lambda pid: set(range(128)), raising=False)
    monkeypatch.setattr(builtins, 'open', fake_open('1600000 100000\n'))
    assert bench.cgroup_cpu_limit() == 16 and bench.host_cores() == 16 and hostio.usable_cpus() == 16
    monkeypatch.setattr(builtins, 'open', fake_open('max 100000\n'))
    assert bench.cgroup_cpu_limit() is None and bench.host_cores() == 128 and hostio.usable_cpus() == 128
    monkeypatch.setattr(builtins, 'open', fake_open('150000 100000\n'))         # 1.5 CPUs -> 2
    assert bench.cgroup_cpu_limit() == 2 and bench.host_cores() == 2
