"""Write golden_gzip.json: SHA-256 and size of the simulated engine's pb200GzipDevice output (tests/sim) for seeded inputs, so
that tests/test_gpu_gzip.py can check that the device writes exactly the same bytes.

    python tests/golden/make_golden_gzip.py
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
sys.path[:0] = [os.path.dirname(TESTS), TESTS, os.path.join(TESTS, 'sim')]

from gzip_inputs import golden_cases  # noqa: E402


def main():
    import sim_engine
    from test_trim_split_reads import SimDevice
    W = sim_engine.load()
    D = SimDevice(W)
    out = {}
    for name, (data, seg, block) in golden_cases().items():
        d = D.upload(np.frombuffer(data, dtype=np.uint8))
        cap = W.gzip_bound(len(data), 1 if seg is None else len(seg) - 1, block)
        buf = D.empty(max(cap, 1), np.uint8)
        total, off = W.pb200_gzip_device(D.ptr(d), len(data), seg, block=block, d_out_ptr=D.ptr(buf), out_cap=cap)
        gz = D.host(D.head(buf, total)).tobytes()
        out[name] = {'n': len(data), 'block': block, 'size': total, 'seg_out': [int(x) for x in off],
                     'sha256': hashlib.sha256(gz).hexdigest()}
        D.free()
    with open(os.path.join(HERE, 'golden_gzip.json'), 'w') as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write('\n')


if __name__ == '__main__':
    main()
