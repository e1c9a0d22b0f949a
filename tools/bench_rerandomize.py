"""Groth16 proof rerandomization on the GPU (b2g_rerandomize_many): proofs per second of one synchronous call.

The work per proof does not depend on the key beyond delta_2, so one key serves: test.zkey, with `--distinct` proofs
(tools/bench_verify.key_test) repeated up to each count.  For each count, the rows and random factors are encoded once and
every call goes straight through the C ABI; one warm-up call grows the context's buffers, then the rate is count over the
best of `--reps` calls (at count 1 the best time is the latency).  A sample of each call's rows is checked against the big-int
model of tests/rerandomize_model.py.  For scale, the same model's rate on one core.

    python tools/bench_rerandomize.py [--counts 1,1024,16384,65536] [--reps 3]
"""
import argparse
import ctypes as C
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from bench_verify import gpu_label, key_test  # noqa: E402
from circom_compat_b200 import Context, release  # noqa: E402
from circom_compat_b200 import _native as N  # noqa: E402
from circom_compat_b200 import verifier as V  # noqa: E402
from oracle import pyref  # noqa: E402
from rerandomize_model import proof_bytes, proof_points, rerandomize_proof  # noqa: E402

R = pyref.R_MOD


def _ptr(a):
    return C.c_void_p(a.ctypes.data)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,1024,16384,65536')
    ap.add_argument('--distinct', type=int, default=256)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--host-proofs', type=int, default=8)
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(',')]
    print(f'# GPU: {gpu_label()}', flush=True)
    ctx = Context(0)
    L = N.lib()
    pk, _, proofs = key_test(ctx, args.distinct)
    vh, m = ctx.vk_handle(pk), len(proofs)
    delta = V.VerifyingKey.from_proving_key(pk).delta_g2
    rng = random.Random(5)

    def model(p, r1, r2):
        return proof_bytes(rerandomize_proof(delta, proof_points(p), r1, r2))

    t0 = time.perf_counter()
    for p in proofs[:args.host_proofs]:
        model(p.data, rng.randrange(1, R), rng.randrange(1, R))
    host_rate = round(args.host_proofs / (time.perf_counter() - t0), 1)
    print(json.dumps({'host_python_rerandomize_proofs_per_s': host_rate, 'model': 'tests/rerandomize_model.py, one core'}), flush=True)
    row = {}
    for count in counts:
        rows = [proofs[k % m].data for k in range(count)]
        fs = [(rng.randrange(1, R), rng.randrange(1, R)) for _ in range(count)]
        data = np.frombuffer(b''.join(rows), dtype=np.uint8).copy()
        r1 = np.frombuffer(b''.join(a.to_bytes(32, 'little') for a, _ in fs), dtype=np.uint8).copy()
        r2 = np.frombuffer(b''.join(b.to_bytes(32, 'little') for _, b in fs), dtype=np.uint8).copy()
        out, ok = np.zeros((count, 256), dtype=np.uint8), np.zeros(count, dtype=np.uint8)
        call = lambda: N.check(L.b2g_rerandomize_many(ctx._h, vh, count, _ptr(data), _ptr(r1), _ptr(r2), _ptr(out), _ptr(ok)))
        call()                                                            # warm-up: buffers
        best = None
        for _ in range(args.reps):
            t0 = time.perf_counter()
            call()
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        assert ok.all(), count
        for i in {0, count - 1, rng.randrange(count)}:
            assert out[i].tobytes() == model(rows[i], *fs[i]), (count, i)
        row[f'rerandomize_proofs_per_s@{count}'] = round(count / best, 1)
        if count == 1:
            row['rerandomize_latency_ms'] = round(best * 1e3, 3)
        print(json.dumps({'count': count, 'best_ms': round(best * 1e3, 3), 'proofs_per_s': round(count / best, 1)}), flush=True)
    print(json.dumps(row), flush=True)
    release(pk)
    ctx.close()


if __name__ == '__main__':
    main()
