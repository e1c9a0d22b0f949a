"""Arkworks-serialized proving keys: serialize_proving_key, and deserialize_proving_key from compressed and from uncompressed
bytes, on whole keys, host parsing included (ark_serialize.py over b2g_points_serialize / b2g_points_deserialize).

Keys: test.zkey, the reference's bench key (complex-circuit-10000-10000.zkey, domain 2^14) and synthetic squaring-chain keys
made by synth.setup on the GPU (--sizes, log2 of the domain; 2^20 holds about 4.2 M G1 and 1 M G2 points).  Every key is
checked to read back bit for bit before it is timed.  A time is the best of --reps calls.  For scale, the big-int model of the
format (tests/ark_key_model.py, one point at a time on the host, as oracle.pyref decodes proofs) is timed on a small sample of
the bench key's compressed points; its rate is stated for that sample and not extrapolated.

    python tools/bench_ark_keys.py [--sizes 16,18,20] [--reps 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from bench_verify import gpu_label  # noqa: E402
from circom_compat_b200 import Context, deserialize_proving_key, read_zkey, serialize_proving_key, synth  # noqa: E402

ARRAYS = ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'delta_g1', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query',
          'b_g2_query', 'l_query', 'h_query')


def points(pk):
    g1 = sum(np.asarray(getattr(pk, n)).size // 8 for n in ARRAYS if n.endswith('g1') or n in ('a_query', 'b_g1_query', 'l_query', 'h_query'))
    g2 = sum(np.asarray(getattr(pk, n)).size // 16 for n in ('beta_g2', 'gamma_g2', 'delta_g2', 'b_g2_query'))
    return g1, g2


def same(a, b):
    return all(np.ascontiguousarray(getattr(a, n), dtype='<u8').tobytes() == getattr(b, n).tobytes() for n in ARRAYS)


def best(fn, reps):
    t, out = float('inf'), None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        t = min(t, time.perf_counter() - t0)
    return t, out


def model_rate(pk, n_g1=64, n_g2=16):
    """points per second of the big-int model decoding compressed points of `pk` (Validate::Yes), on that sample"""
    import ark_key_model as M
    from circom_compat_b200.verifier import _g1_from_words, _g2_from_words
    g1 = [_g1_from_words(r) for r in pk.a_query[:n_g1]]
    g2 = [_g2_from_words(r) for r in pk.b_g2_query[:4 * n_g2] if r.any()][:n_g2]
    raw = [(M.point_bytes(p, False, True), False) for p in g1] + [(M.point_bytes(q, True, True), True) for q in g2]
    t0 = time.perf_counter()
    for b, g in raw:
        M.decode_point(b, g, True)
    dt = time.perf_counter() - t0
    return {'sample_g1': len(g1), 'sample_g2': len(g2), 'seconds': dt, 'points_per_s': len(raw) / dt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='16,18,20')
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    label = gpu_label()
    ctx = Context(0)
    keys = [('test.zkey', lambda: read_zkey(open(os.path.join(ROOT, 'tests', 'golden', 'test.zkey'), 'rb').read())[0]),
            ('bench key 2^14', lambda: read_zkey(open(os.path.join(ROOT, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'), 'rb').read())[0])]
    keys += [(f'synthetic 2^{s}', lambda s=s: synth.setup(ctx, synth.chain_circuit(1 << s))[0]) for s in map(int, args.sizes.split(','))]
    rows = []
    for name, make in keys:
        pk = make()
        g1, g2 = points(pk)
        row = {'key': name, 'g1_points': g1, 'g2_points': g2}
        for compress, form in ((True, 'compressed'), (False, 'uncompressed')):
            data = serialize_proving_key(pk, compress, ctx)                  # warm-up, and the bytes to read back
            assert same(pk, deserialize_proving_key(data, compress, ctx)), (name, form)
            t_ser, _ = best(lambda: serialize_proving_key(pk, compress, ctx), args.reps)
            t_de, _ = best(lambda: deserialize_proving_key(data, compress, ctx), args.reps)
            row[f'{form}_bytes'] = len(data)
            row[f'serialize_{form}_s'] = t_ser
            row[f'deserialize_{form}_s'] = t_de
            row[f'deserialize_{form}_points_per_s'] = (g1 + g2) / t_de
        rows.append(row)
        print(json.dumps(row), flush=True)
        if name.startswith('bench'):
            model = model_rate(pk)
    print(json.dumps({'model': model}))
    print(f"\n{label}; best of {args.reps}; wall time per whole key, host parsing included\n")
    print('| key | G1 + G2 points | serialize (compressed) | deserialize compressed | deserialize uncompressed |')
    print('|---|---|---|---|---|')
    for r in rows:
        n = r['g1_points'] + r['g2_points']
        print(f"| {r['key']} | {r['g1_points']:,} + {r['g2_points']:,} | {r['serialize_compressed_s'] * 1e3:.1f} ms | "
              f"{r['deserialize_compressed_s'] * 1e3:.1f} ms ({n / r['deserialize_compressed_s'] / 1e6:.2f} M points/s) | "
              f"{r['deserialize_uncompressed_s'] * 1e3:.1f} ms ({n / r['deserialize_uncompressed_s'] / 1e6:.2f} M points/s) |")
    print(f"\nbig-int model (host, one point at a time): {model['points_per_s']:.0f} points/s measured on "
          f"{model['sample_g1']} G1 + {model['sample_g2']} G2 compressed points of the bench key")
    ctx.close()


if __name__ == '__main__':
    main()
