"""Per-proof verdicts under many verifying keys: one b2g_verify_batch_keys_locate call against a loop of
b2g_verify_batch_locate per key, and against the recipe that came before it (b2g_verify_batch_keys, then
b2g_verify_batch_locate on every key whose verdict is 0).

Keys and proofs come from bench_verify_keys.make_keys (known discrete logs, made on the device); batch k is checked under key
k mod the number of distinct keys, as there.  Every workload is timed in four cases: all valid, one invalid proof in the whole
call, one invalid proof per key, and 1 % of the proofs invalid (A negated, spread over the call).  Inputs, proofs and weights
are encoded once per case; all arms go through the C ABI and their verdicts are checked against the planted set.  Each
repetition runs the arms in turn; a time is the best of --reps calls (the two per-key loops: of --loop-reps).

    python tools/bench_verify_keys_locate.py [--reps 3] [--loop-reps 3] [--inputs 1,100] [--shapes 16x16,256x16,256x256,1024x1]
"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_verify import gpu_label  # noqa: E402
from bench_verify_keys import _ptr, encode, make_keys  # noqa: E402
from circom_compat_b200 import Context, release  # noqa: E402
from circom_compat_b200 import _native as N  # noqa: E402
from circom_compat_b200 import verifier as V  # noqa: E402

P = V.P
SHAPES = [(16, 16), (256, 16), (256, 256), (1024, 1)]
CASES = ('all valid', 'one invalid', 'one invalid per key', '1% invalid')


def _negate_a(rows, i):
    """A -> -A in proof row i of a (count x 256 B) array: y -> p - y"""
    y = int.from_bytes(rows[256 * i + 32:256 * i + 64].tobytes(), 'little')
    rows[256 * i + 32:256 * i + 64] = np.frombuffer(((P - y) % P).to_bytes(32, 'little'), dtype=np.uint8)


def plant(batches, case, rng):
    """the proofs of `case` made invalid in place; returns the set of (batch, proof) pairs"""
    counts = [m for _, m, _, _, _ in batches]
    total = sum(counts)
    if case == 'all valid':
        bad = set()
    elif case == 'one invalid':
        bad = {(len(counts) // 2, counts[len(counts) // 2] // 2)}
    elif case == 'one invalid per key':
        bad = {(k, rng.randrange(m)) for k, m in enumerate(counts)}
    else:
        flat = [(k, i) for k, m in enumerate(counts) for i in range(m)]
        bad = set(rng.sample(flat, max(1, total // 100)))
    for k, i in bad:
        _negate_a(batches[k][3], i)
    return bad


def measure(ctx, keys, handles, counts, case, reps, loop_reps, seed):
    L = N.lib()
    batches = encode(keys, counts)
    bad = plant(batches, case, random.Random(seed))
    want = [[(k, i) not in bad for i in range(m)] for k, m in enumerate(counts)]
    table = (N.KeyBatch * len(batches))(*[N.KeyBatch(handles[key].value, m, 0, _ptr(pub), _ptr(pr), _ptr(w))
                                          for key, m, pub, pr, w in batches])
    total = sum(counts)
    verdicts, per_key = np.zeros(total, dtype=np.uint8), np.zeros(len(batches), dtype=np.uint8)
    outs = [np.zeros(m, dtype=np.uint8) for m in counts]
    flat_want = [v for w in want for v in w]

    def keyed():
        N.check(L.b2g_verify_batch_keys_locate(ctx._h, len(batches), table, _ptr(verdicts)))
        assert verdicts.tolist() == flat_want

    def loop():
        for (key, m, pub, pr, w), out, wk in zip(batches, outs, want):
            N.check(L.b2g_verify_batch_locate(ctx._h, handles[key], m, _ptr(pub), _ptr(pr), _ptr(w), _ptr(out)))
            assert out.tolist() == wk

    def old():
        N.check(L.b2g_verify_batch_keys(ctx._h, len(batches), table, _ptr(per_key)))
        for (key, m, pub, pr, w), out, wk, ok in zip(batches, outs, want, per_key):
            if not ok:
                N.check(L.b2g_verify_batch_locate(ctx._h, handles[key], m, _ptr(pub), _ptr(pr), _ptr(w), _ptr(out)))
                assert out.tolist() == wk
            else:
                assert all(wk)

    arms = (('keyed', keyed, reps), ('loop', loop, loop_reps), ('keys_then_locate', old, loop_reps))
    keyed()                                                        # warm-up (buffers) and check
    best = {}
    for r in range(max(reps, loop_reps)):
        for label, fn, n in arms:
            if r >= n:
                continue
            t0 = time.perf_counter()
            fn()
            dt = time.perf_counter() - t0
            best[label] = min(best.get(label, dt), dt)
    row = {'keys': len(counts), 'proofs': total, 'invalid': len(bad)}
    for label, _, _ in arms:
        row[f'{label}_ms'] = round(best[label] * 1e3, 2)
    row['keyed_speedup_over_loop'] = round(best['loop'] / best['keyed'], 1)
    row['keyed_speedup_over_keys_then_locate'] = round(best['keys_then_locate'] / best['keyed'], 1)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--loop-reps', type=int, default=3)
    ap.add_argument('--inputs', default='1,100')
    ap.add_argument('--shapes', default=','.join(f'{k}x{m}' for k, m in SHAPES))
    args = ap.parse_args()
    shapes = [tuple(int(v) for v in s.split('x')) for s in args.shapes.split(',')]
    ctx = Context(0)
    print(f'# GPU: {gpu_label()}', flush=True)
    for n_public in (int(x) for x in args.inputs.split(',')):
        keys = make_keys(ctx, 256 if n_public < 16 else 16, n_public, 16, 7 + n_public)
        handles = [ctx.vk_handle(vk) for vk, _, _ in keys]
        for k, m in shapes:
            for c, case in enumerate(CASES):
                row = {'n_public': n_public, 'workload': f'{k} x {m}', 'case': case,
                       **measure(ctx, keys, handles, [m] * k, case, args.reps, args.loop_reps, 100 * k + m + c)}
                print(json.dumps(row), flush=True)
        for vk, _, _ in keys:
            release(vk)
    ctx.close()


if __name__ == '__main__':
    main()
