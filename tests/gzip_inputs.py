"""Inputs and checks shared by the gzip tests (pb200GzipDevice): the edge set, a seeded ONT-like FASTQ model, and a walk over
the members of a gzip file.  Used by test_gzip_device.py (simulated engine), test_gpu_gzip.py and
golden/make_golden_gzip.py."""
import uuid
import zlib

import numpy as np

BLOCK = 4096          # the smallest block the engine takes: edge cases stay small, and many members run through few bytes


def ont_fastq(n_bytes, seed=0):
    """ONT-like FASTQ of about n_bytes: UUID names with runid / read / ch / start_time fields, log-normal read lengths around
    5 kb, random bases, and qualities as runs (geometric lengths) of a random walk folded into Phred 2..40"""
    rng = np.random.default_rng(seed)
    run = ''.join('%x' % v for v in rng.integers(0, 16, 40))
    out, size = [], 0
    while size < n_bytes:
        n = int(min(max(rng.lognormal(np.log(5000), 0.6), 200), 60000))
        name = '%s runid=%s read=%d ch=%d start_time=2026-01-%02dT%02d:%02d:%02dZ' % (
            uuid.UUID(bytes=rng.bytes(16), version=4), run, int(rng.integers(1, 99999)), int(rng.integers(1, 513)),
            int(rng.integers(1, 29)), int(rng.integers(0, 24)), int(rng.integers(0, 60)), int(rng.integers(0, 60)))
        seq = np.frombuffer(b'ACGT', dtype=np.uint8)[rng.integers(0, 4, n)]
        walk = np.abs(((np.cumsum(rng.integers(-4, 5, n)) + 20) % 76) - 38) + 2
        qual = np.repeat(walk, rng.geometric(0.35, n))[:n].astype(np.uint8) + 33
        rec = b'@' + name.encode() + b'\n' + seq.tobytes() + b'\n+\n' + qual.tobytes() + b'\n'
        out.append(rec)
        size += len(rec)
    return b''.join(out)


def edge_inputs(block=BLOCK):
    """{name: bytes}: the lengths around the block size, runs, every byte value, periods at the distance limit, random bytes"""
    rng = np.random.default_rng(7)
    period = lambda p, n: np.resize(rng.integers(0, 256, p, dtype=np.uint8), n).tobytes()      # noqa: E731
    return {
        'empty': b'', 'one': b'A', 'two': b'AC', 'three': b'ACG',
        'block_minus_1': rng.integers(65, 69, block - 1, dtype=np.uint8).tobytes(),
        'block': rng.integers(65, 69, block, dtype=np.uint8).tobytes(),
        'block_plus_1': rng.integers(65, 69, block + 1, dtype=np.uint8).tobytes(),
        'several_blocks': ont_fastq(5 * block + 123, 3)[:5 * block + 123],
        'zeros': bytes(3 * block + 17),
        'every_byte': bytes(range(256)) * 40 + bytes(range(255, -1, -1)) * 3,
        'period_32768': period(32768, 3 * 32768 + 100),
        'period_32769': period(32769, 3 * 32769 + 100),
        'random': rng.integers(0, 256, 4 * block, dtype=np.uint8).tobytes(),
    }


def segments_of(lengths):
    """seg_off of consecutive segments with these lengths"""
    return [0] + np.cumsum(lengths).astype(np.int64).tolist()


def members(gz):
    """the members of a gzip file: [(compressed bytes, decompressed bytes)], walked with zlib.decompressobj(31) and its
    unused_data (fed in 64 KB pieces, so that a file of many members is walked in linear time)"""
    out, pos = [], 0
    while pos < len(gz):
        d, start, plain = zlib.decompressobj(31), pos, []
        while not d.eof:
            piece = gz[pos:pos + 65536]
            assert piece, 'truncated member'
            plain.append(d.decompress(piece))
            pos += len(piece)
        pos -= len(d.unused_data)
        out.append((gz[start:pos], b''.join(plain)))
    return out


HEADER = bytes([0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3])


def check_file(gz, plain, block):
    """gz decompresses to plain, as ceil(len / block) members that each start with the header and hold block bytes (the last
    one the rest)"""
    ms = members(gz)
    assert len(ms) == (len(plain) + block - 1) // block
    assert b''.join(p for _, p in ms) == plain
    for k, (c, p) in enumerate(ms):
        assert c[:10] == HEADER
        assert len(p) == min(block, len(plain) - k * block)


def zlib_level_bytes(data, block, level):
    """bytes of zlib at `level`, one gzip member per block"""
    total = 0
    for i in range(0, len(data), block):
        c = zlib.compressobj(level, zlib.DEFLATED, 31)
        total += len(c.compress(data[i:i + block]) + c.flush())
    return total


def golden_cases():
    """{name: (data, seg_off or None, block)} of golden_gzip.json: the edge set, the ONT model at the default block as one
    file and as 48 segments, and one input at each other block size"""
    cases = {'edge_' + k: (v, None, BLOCK) for k, v in edge_inputs().items()}
    big = ont_fastq(2_000_000, 21)
    cases['ont_default_block'] = (big, None, 0)
    cuts = np.sort(np.random.default_rng(22).integers(0, len(big), 47)).tolist()
    cases['ont_48_segments'] = (big, [0] + cuts + [len(big)], 0)
    for block in (32768, 131072):
        cases['ont_block_%d' % block] = (big[:400_000], None, block)
    return cases
