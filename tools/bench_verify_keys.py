"""Batches under many verifying keys: one b2g_verify_batch_keys call against a loop of b2g_verify_batch per key, and against
one b2g_verify_batch over as many proofs of a single key (the ceiling).

Keys and proofs are made with known discrete logs on the device (Context.fixed_base_g1 / g2).  The 1-input workloads use up
to 256 distinct keys and the 100-input ones up to 16 (a 100-input key holds 51 MB of window tables); batch k is checked under
key k mod that number, which leaves every per-key stage (tails, IC products) as it is for distinct keys.  Each distinct key has
16 distinct valid proofs, cycled.  Inputs, proofs and weights are encoded once; all three arms go through the C ABI.  Each
repetition runs the three arms in turn; a rate is the proofs over the best of --reps calls.

    python tools/bench_verify_keys.py [--reps 3] [--inputs 1,100]
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

from bench_verify import gpu_label  # noqa: E402
from circom_compat_b200 import Context, Proof, release  # noqa: E402
from circom_compat_b200 import _native as N  # noqa: E402
from circom_compat_b200 import verifier as V  # noqa: E402
from oracle import pyref as o  # noqa: E402

P, R = V.P, o.R_MOD
RINV = pow(1 << 256, -1, P)
GRID = [(k, m) for k in (1, 16, 256, 1024) for m in (1, 16, 256) if k * m <= 65536]


def _ptr(a):
    return a.ctypes.data if a is not None and a.size else None


def _limbs(ks):
    return np.frombuffer(b''.join(k.to_bytes(32, 'little') for k in ks), dtype='<u8').copy()


def _canon(rows):
    raw, w = np.ascontiguousarray(rows).tobytes(), rows.shape[1] // 4
    v = [int.from_bytes(raw[i:i + 32], 'little') * RINV % P for i in range(0, len(raw), 32)]
    return [v[k * w:(k + 1) * w] for k in range(rows.shape[0])]


def make_keys(ctx, n_keys, n_public, n_proofs, seed):
    """n_keys (vk, public-input bytes per proof, proof bytes per proof) with n_proofs valid proofs each"""
    rng = random.Random(seed)
    plan, s1, s2 = [], [], []
    for _ in range(n_keys):
        al, be, ga, de = (rng.randrange(1, R) for _ in range(4))
        ic = [rng.randrange(1, R) for _ in range(n_public + 1)]
        rows = []
        for _ in range(n_proofs):
            xs = [rng.randrange(R) for _ in range(n_public)]
            a, b = rng.randrange(1, R), rng.randrange(1, R)
            prep = (ic[0] + sum(x * k for x, k in zip(xs, ic[1:]))) % R
            rows.append((xs, a, b, (a * b - al * be - prep * ga) * pow(de, -1, R) % R))
        plan.append(rows)
        s1 += [al] + ic + [v for _, a, _, c in rows for v in (a, c)]
        s2 += [be, ga, de] + [b for _, _, b, _ in rows]
    g1 = [tuple(p) for p in _canon(ctx.fixed_base_g1(_limbs(s1)))]
    g2 = [((q[0], q[1]), (q[2], q[3])) for q in _canon(ctx.fixed_base_g2(_limbs(s2)))]
    out, i1, i2 = [], 0, 0
    for rows in plan:
        vk = V.VerifyingKey(g1[i1], g2[i2], g2[i2 + 1], g2[i2 + 2], g1[i1 + 1:i1 + 2 + n_public])
        i1 += 2 + n_public
        i2 += 3
        pubs, proofs = [], []
        for xs, _, _, _ in rows:
            a, b, c = g1[i1], g2[i2], g1[i1 + 1]
            vals = list(a) + [b[0][0], b[0][1], b[1][0], b[1][1]] + list(c)
            proofs.append(Proof(b''.join(int(v).to_bytes(32, 'little') for v in vals)).data)
            pubs.append(b''.join(int(x).to_bytes(32, 'little') for x in xs))
            i1 += 2
            i2 += 1
        out.append((vk, pubs, proofs))
    return out


def encode(keys, counts):
    """per batch (key index, count, public inputs, proofs, weights) as arrays; batch k under key k mod len(keys)"""
    out = []
    for k, m in enumerate(counts):
        key = k % len(keys)
        _, pubs, proofs = keys[key]
        pub = b''.join(pubs[i % len(pubs)] for i in range(m))
        out.append((key, m, np.frombuffer(pub, dtype=np.uint8).copy() if pub else None,
                    np.frombuffer(b''.join(proofs[i % len(proofs)] for i in range(m)), dtype=np.uint8).copy(),
                    np.frombuffer(b''.join((secrets.randbits(128) | 1).to_bytes(16, 'little') for _ in range(m)), dtype=np.uint8).copy()))
    return out


def measure(ctx, keys, handles, counts, reps):
    L = N.lib()
    batches = encode(keys, counts)
    table = (N.KeyBatch * len(batches))(*[N.KeyBatch(handles[key].value, m, 0, _ptr(pub), _ptr(pr), _ptr(w))
                                          for key, m, pub, pr, w in batches])
    verdicts, one = np.zeros(len(batches), dtype=np.uint8), np.zeros(1, dtype=np.uint8)
    total = sum(counts)
    ceiling = encode(keys[:1], [total])[0]

    def keyed():
        N.check(L.b2g_verify_batch_keys(ctx._h, len(batches), table, _ptr(verdicts)))
        assert verdicts.all()

    def loop():
        for key, m, pub, pr, w in batches:
            N.check(L.b2g_verify_batch(ctx._h, handles[key], m, _ptr(pub), _ptr(pr), _ptr(w), _ptr(one)))
            assert one[0] == 1

    def single():
        _, m, pub, pr, w = ceiling
        N.check(L.b2g_verify_batch(ctx._h, handles[0], m, _ptr(pub), _ptr(pr), _ptr(w), _ptr(one)))
        assert one[0] == 1

    arms = (('keyed', keyed), ('loop', loop), ('ceiling', single))
    for _, fn in arms:                                             # warm-up (buffers) and check
        fn()
    best = {}
    for _ in range(reps):
        for label, fn in arms:
            t0 = time.perf_counter()
            fn()
            dt = time.perf_counter() - t0
            best[label] = min(best.get(label, dt), dt)
    row = {'keys': len(counts), 'proofs': total}
    for label, _ in arms:
        row[f'{label}_ms'] = round(best[label] * 1e3, 2)
        row[f'{label}_proofs_per_s'] = round(total / best[label], 1)
    row['keyed_speedup_over_loop'] = round(best['loop'] / best['keyed'], 2)
    row['keyed_over_ceiling'] = round(best['keyed'] / best['ceiling'], 2)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--inputs', default='1,100')
    args = ap.parse_args()
    ctx = Context(0)
    print(f'# GPU: {gpu_label()}', flush=True)
    for n_public in (int(x) for x in args.inputs.split(',')):
        keys = make_keys(ctx, 256 if n_public < 16 else 16, n_public, 16, 7 + n_public)
        handles = [ctx.vk_handle(vk) for vk, _, _ in keys]
        work = [(f'{k} x {m}', [m] * k) for k, m in GRID]
        work.append(('16384 + 255 x 16', [16384] + [16] * 255))
        for name, counts in work:
            row = {'n_public': n_public, 'workload': name, **measure(ctx, keys, handles, counts, args.reps)}
            print(json.dumps(row), flush=True)
        for vk, _, _ in keys:
            release(vk)
    ctx.close()


if __name__ == '__main__':
    main()
