"""Per-proof verdicts from the grouped batch check (b2g_verify_batch_locate) against today's recipe, one batch verdict
(b2g_verify_batch) followed by b2g_verify_many when it fails, and against b2g_verify_many alone, on the GPU.

Keys and proofs as tools/bench_verify.py (test, complex, synth100).  Scenarios: every proof valid; one invalid proof at a
random position; 1 % invalid proofs spread at random; one invalid proof in every group of 64.  An invalid proof is a valid
one with A negated.  For each key, count and scenario, the public inputs, proofs and weights are encoded once and every
call goes straight through the C ABI.  Each repetition runs the three arms in turn; the time of an arm is its best over the
repetitions, in milliseconds.  Every arm's verdicts are checked against the scenario's.

    python tools/bench_verify_locate.py [--counts 1,1024,16384,65536] [--keys test,complex,synth100] [--reps 3]
"""
import argparse
import ctypes as C
import json
import os
import random
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
from circom_compat_b200 import verifier as V  # noqa: E402

GROUP = 64


def _ptr(a):
    return C.c_void_p(a.ctypes.data) if a is not None and a.size else None


def _bad_positions(scenario, count, rng):
    if scenario == 'valid':
        return set()
    if scenario == 'one_bad':
        return {rng.randrange(count)}
    if scenario == 'one_percent':
        return set(rng.sample(range(count), max(1, count // 100)))
    return {g + rng.randrange(min(GROUP, count - g)) for g in range(0, count, GROUP)}     # one per group


def _negate_a(row: bytes) -> bytes:
    y = int.from_bytes(row[32:64], 'little')
    return row[:32] + ((V.P - y) % V.P).to_bytes(32, 'little') + row[64:]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,1024,16384,65536')
    ap.add_argument('--keys', default='test,complex,synth100')
    ap.add_argument('--scenarios', default='valid,one_bad,one_percent,one_per_group')
    ap.add_argument('--distinct', type=int, default=256)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(',')]
    ctx = Context(0)
    L = N.lib()
    print(f'# GPU: {gpu_label()}', flush=True)
    makers = {'test': key_test, 'complex': key_complex, 'synth100': lambda c, n: key_synth100(c, min(n, 64))}
    rng = random.Random(7)
    for name in args.keys.split(','):
        key, inputs, proofs = makers[name](ctx, args.distinct)
        m, vh = len(proofs), ctx.vk_handle(key)
        pub1 = [b''.join(int(x).to_bytes(32, 'little') for x in xs) for xs in inputs]
        for scenario in args.scenarios.split(','):
            row = {'key': name, 'n_public': len(inputs[0]), 'scenario': scenario}
            for count in counts:
                bad = _bad_positions(scenario, count, rng)
                pub = np.frombuffer(b''.join(pub1[k % m] for k in range(count)), dtype=np.uint8).copy() if inputs[0] else None
                data = np.frombuffer(b''.join(_negate_a(proofs[k % m].data) if k in bad else proofs[k % m].data for k in range(count)),
                                     dtype=np.uint8).copy()
                w = np.frombuffer(b''.join((secrets.randbits(128) | 1).to_bytes(16, 'little') for _ in range(count)), dtype=np.uint8).copy()
                want = np.array([k not in bad for k in range(count)], dtype=np.uint8)
                out = {a: np.zeros(count, dtype=np.uint8) for a in ('locate', 'recipe', 'many')}
                one = np.zeros(1, dtype=np.uint8)

                def locate():
                    N.check(L.b2g_verify_batch_locate(ctx._h, vh, count, _ptr(pub), _ptr(data), _ptr(w), _ptr(out['locate'])))

                def recipe():
                    N.check(L.b2g_verify_batch(ctx._h, vh, count, _ptr(pub), _ptr(data), _ptr(w), _ptr(one)))
                    if one[0]:
                        out['recipe'][:] = 1
                    else:
                        N.check(L.b2g_verify_many(ctx._h, vh, count, _ptr(pub), _ptr(data), _ptr(out['recipe'])))

                def many():
                    N.check(L.b2g_verify_many(ctx._h, vh, count, _ptr(pub), _ptr(data), _ptr(out['many'])))

                arms = (('locate', locate), ('recipe', recipe), ('many', many))
                for label, fn in arms:                                    # warm-up (buffers) and check
                    fn()
                    assert (out[label] == want).all(), (name, scenario, count, label)
                best = {}
                for _ in range(args.reps):
                    for label, fn in arms:
                        t0 = time.perf_counter()
                        fn()
                        dt = time.perf_counter() - t0
                        best[label] = min(best.get(label, dt), dt)
                for label, _ in arms:
                    row[f'{label}_ms@{count}'] = round(best[label] * 1e3, 3)
            print(json.dumps(row), flush=True)
        release(key)
    ctx.close()


if __name__ == '__main__':
    main()
