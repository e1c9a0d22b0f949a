"""Compressed proofs (arkworks' 128-byte serialize_compressed) decoded and verified on the GPU, against the same proofs given
as 256-byte rows.

Keys and proofs as tools/bench_verify.py (test, complex, synth100).  For each key and count, the public inputs, the 256-byte
rows, the compressed rows and the weights are encoded once, and every call goes straight through the C ABI.  Each repetition
runs, alternating: b2g_proofs_decompress alone, b2g_verify_many then b2g_verify_many_compressed, b2g_verify_batch then
b2g_verify_batch_compressed.  The rate is count over the best call time; at count 1 the best time is the latency.  For
scale, the host decode rate of the oracle's big-int decoder (oracle.pyref.decompress_proof, no G2 check) on one core.

    python tools/bench_verify_compressed.py [--counts 1,1024,16384,65536] [--keys test,complex,synth100] [--reps 3]
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
from circom_compat_b200 import Context, release  # noqa: E402
from circom_compat_b200 import _native as N  # noqa: E402
from circom_compat_b200 import ethereum as eth  # noqa: E402
from oracle import pyref  # noqa: E402


def _ptr(a):
    return C.c_void_p(a.ctypes.data) if a is not None and a.size else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,1024,16384,65536')
    ap.add_argument('--keys', default='test,complex,synth100')
    ap.add_argument('--distinct', type=int, default=256)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(',')]
    ctx = Context(0)
    L = N.lib()
    print(f'# GPU: {gpu_label()}', flush=True)
    makers = {'test': key_test, 'complex': key_complex, 'synth100': lambda c, n: key_synth100(c, min(n, 64))}
    host_rate = None
    for name in args.keys.split(','):
        key, inputs, proofs = makers[name](ctx, args.distinct)
        m, vh = len(proofs), ctx.vk_handle(key)
        pub1 = [b''.join(int(x).to_bytes(32, 'little') for x in xs) for xs in inputs]
        comp1 = [eth.serialize_compressed(eth.Proof.from_proof(p)) for p in proofs]
        if host_rate is None:
            t0 = time.perf_counter()
            for blob in comp1:
                pyref.decompress_proof(blob)
            host_rate = round(m / (time.perf_counter() - t0), 1)
            print(json.dumps({'host_python_decompress_proofs_per_s': host_rate, 'decoder': 'oracle.pyref.decompress_proof, one core, no G2 check'}), flush=True)
        row = {'key': name, 'n_public': len(inputs[0])}
        for count in counts:
            pub = np.frombuffer(b''.join(pub1[k % m] for k in range(count)), dtype=np.uint8).copy() if inputs[0] else None
            data = np.frombuffer(b''.join(proofs[k % m].data for k in range(count)), dtype=np.uint8).copy()
            comp = np.frombuffer(b''.join(comp1[k % m] for k in range(count)), dtype=np.uint8).copy()
            w = np.frombuffer(b''.join((secrets.randbits(128) | 1).to_bytes(16, 'little') for _ in range(count)), dtype=np.uint8).copy()
            verdicts, one = np.zeros(count, dtype=np.uint8), np.zeros(1, dtype=np.uint8)
            rows, ok = np.zeros(count * 256, dtype=np.uint8), np.zeros(count, dtype=np.uint8)
            calls = {
                'decompress': lambda: N.check(L.b2g_proofs_decompress(ctx._h, count, _ptr(comp), _ptr(rows), _ptr(ok))),
                'many': lambda: N.check(L.b2g_verify_many(ctx._h, vh, count, _ptr(pub), _ptr(data), _ptr(verdicts))),
                'many_compressed': lambda: N.check(L.b2g_verify_many_compressed(ctx._h, vh, count, _ptr(pub), _ptr(comp), _ptr(verdicts))),
                'batch': lambda: N.check(L.b2g_verify_batch(ctx._h, vh, count, _ptr(pub), _ptr(data), _ptr(w), _ptr(one))),
                'batch_compressed': lambda: N.check(L.b2g_verify_batch_compressed(ctx._h, vh, count, _ptr(pub), _ptr(comp), _ptr(w), _ptr(one))),
            }
            calls['decompress']()                                        # warm-up (buffers) and checks
            assert ok.all() and rows.tobytes() == data.tobytes(), (name, count)
            for label in ('many_compressed', 'batch_compressed'):
                verdicts[:] = 0; one[:] = 0
                calls[label]()
                assert (one[0] == 1) if label.startswith('batch') else verdicts.all(), (name, count, label)
            calls['many'](); calls['batch']()
            best = {label: None for label in calls}
            for _ in range(args.reps):
                for label, fn in calls.items():
                    t0 = time.perf_counter()
                    fn()
                    dt = time.perf_counter() - t0
                    best[label] = dt if best[label] is None else min(best[label], dt)
            for label, dt in best.items():
                row[f'{label}_proofs_per_s@{count}'] = round(count / dt, 1)
                if count == 1:
                    row[f'{label}_latency_ms'] = round(dt * 1e3, 3)
        print(json.dumps(row), flush=True)
        release(key)
    ctx.close()


if __name__ == '__main__':
    main()
