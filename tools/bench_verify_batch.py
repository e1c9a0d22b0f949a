"""One batch verdict (b2g_verify_batch) against one verdict per proof (b2g_verify_many) on the GPU.

Keys and proofs as tools/bench_verify.py (test, complex, synth100).  For each key and count, the public inputs, proofs and
weights are encoded once and both calls go straight through the C ABI, so Python encoding (which bounds the 100-input
key's verify_many rate) is left out of both.  Each repetition runs verify_batch then verify_many, alternating; the rate is
count over the best call time, and at count 1 the best time is the latency.

    python tools/bench_verify_batch.py [--counts 1,1024,16384,65536] [--keys test,complex,synth100] [--reps 3]
"""
import argparse
import ctypes as C
import json
import os
import secrets
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_verify import gpu_label, key_complex, key_synth100, key_test  # noqa: E402
from circom_compat_b200 import Context, Groth16, release  # noqa: E402
from circom_compat_b200 import _native as N  # noqa: E402


def _ptr(a):
    return C.c_void_p(a.ctypes.data) if a is not None and a.size else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,16,256,1024,4096,16384,65536')
    ap.add_argument('--keys', default='test,complex,synth100')
    ap.add_argument('--distinct', type=int, default=256)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(',')]
    ctx = Context(0)
    L = N.lib()
    print(f'# GPU: {gpu_label()}', flush=True)
    makers = {'test': key_test, 'complex': key_complex, 'synth100': lambda c, n: key_synth100(c, min(n, 64))}
    for name in args.keys.split(','):
        key, inputs, proofs = makers[name](ctx, args.distinct)
        m, vh = len(proofs), ctx.vk_handle(key)
        pub1 = [b''.join(int(x).to_bytes(32, 'little') for x in xs) for xs in inputs]
        row = {'key': name, 'n_public': len(inputs[0])}
        for count in counts:
            pub = np.frombuffer(b''.join(pub1[k % m] for k in range(count)), dtype=np.uint8).copy() if inputs[0] else None
            data = np.frombuffer(b''.join(proofs[k % m].data for k in range(count)), dtype=np.uint8).copy()
            w = np.frombuffer(b''.join((secrets.randbits(128) | 1).to_bytes(16, 'little') for _ in range(count)), dtype=np.uint8).copy()
            verdicts, one = np.zeros(count, dtype=np.uint8), np.zeros(1, dtype=np.uint8)
            batch = lambda: N.check(L.b2g_verify_batch(ctx._h, vh, count, _ptr(pub), _ptr(data), _ptr(w), _ptr(one)))
            many = lambda: N.check(L.b2g_verify_many(ctx._h, vh, count, _ptr(pub), _ptr(data), _ptr(verdicts)))
            batch(); many()                                               # warm-up (buffers) and check
            assert one[0] == 1 and verdicts.all(), (name, count)
            best = {'batch': None, 'many': None}
            for _ in range(args.reps):
                for label, fn in (('batch', batch), ('many', many)):
                    t0 = time.perf_counter()
                    fn()
                    dt = time.perf_counter() - t0
                    best[label] = dt if best[label] is None else min(best[label], dt)
            row[f'batch_proofs_per_s@{count}'] = round(count / best['batch'], 1)
            row[f'many_proofs_per_s@{count}'] = round(count / best['many'], 1)
            if count == 1:
                row['batch_latency_ms'] = round(best['batch'] * 1e3, 3)
                row['many_latency_ms'] = round(best['many'] * 1e3, 3)
        # the Python call, encoding included, at the largest count
        count = counts[-1]
        xs, ps = [inputs[k % m] for k in range(count)], [proofs[k % m] for k in range(count)]
        t0 = time.perf_counter()
        assert Groth16.verify_batch(key, xs, ps, ctx)
        row[f'python_verify_batch_proofs_per_s@{count}'] = round(count / (time.perf_counter() - t0), 1)
        print(json.dumps(row), flush=True)
        release(key)
    ctx.close()


if __name__ == '__main__':
    main()
