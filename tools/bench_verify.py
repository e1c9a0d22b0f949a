"""Batched Groth16 verification rate on the GPU (Groth16.verify_many / b2g_verify_many) against the host verifier.

For each key it proves (or, for the synthetic key, constructs) a few hundred distinct valid proofs, tiles them to each
count, and reports verified proofs/s of one synchronous verify_many call (best of --reps, after one warm-up call at that
count).  Host rates, one core: the C++ mirror's verify_with_processed_vk (host/ark_circom_verifier.hpp, timed by
groth16_bench's B2G_VERIFY_MANY mode on the bench key, whose witnesses it can build) and the Python verifier.  Keys:
  test       tests/golden/test.zkey
  complex    the reference's complex-circuit-10000-10000 bench key (2^14)
  synth100   a synthetic key with 100 public inputs (known discrete logs, proofs solved for C)

    python tools/bench_verify.py [--counts 1,64,1024,16384,65536] [--keys test,complex,synth100]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from circom_compat_b200 import Context, Groth16, Proof, fr_to_mont, read_zkey, release  # noqa: E402
from circom_compat_b200 import verifier as V  # noqa: E402
from oracle import pyref as o  # noqa: E402

R = o.R_MOD
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def _proof_bytes(a, b, c):
    vals = list(a) + [b[0][0], b[0][1], b[1][0], b[1][1]] + list(c)
    return Proof(b''.join(int(v).to_bytes(32, 'little') for v in vals))


def key_test(ctx, n):
    pk, cm = read_zkey(open(os.path.join(GOLDEN, 'test.zkey'), 'rb').read())
    g = json.load(open(os.path.join(GOLDEN, 'golden_vectors.json')))['test_zkey']
    w = [int(x) for x in g['witness']]
    rng = random.Random(1)
    proofs = Groth16.create_proofs(pk, [(rng.randrange(R), rng.randrange(R)) for _ in range(n)], cm, [fr_to_mont(w)] * n, ctx)
    release(cm)
    return pk, [w[1:pk.n_public + 1]] * n, proofs


def key_complex(ctx, n):
    pk, cm = read_zkey(open(os.path.join(GOLDEN, 'complex-circuit-10000-10000.zkey'), 'rb').read())
    rng = random.Random(2)
    ws = [o.chain_witness(pk.n_vars, 3 + k) for k in range(n)]
    proofs = Groth16.create_proofs(pk, [(rng.randrange(R), rng.randrange(R)) for _ in ws], cm, [fr_to_mont(w) for w in ws], ctx)
    release(cm)
    return pk, [list(w[1:pk.n_public + 1]) for w in ws], proofs


def key_synth100(ctx, n, n_public=100):
    rng = random.Random(3)
    al, be, ga, de = (rng.randrange(1, R) for _ in range(4))
    ic = [rng.randrange(1, R) for _ in range(n_public + 1)]
    g1 = lambda k: o.G1.mul(o.G1_GEN, k)
    g2 = lambda k: o.G2.mul(o.G2_GEN, k)
    vk = V.VerifyingKey(g1(al), g2(be), g2(ga), g2(de), [g1(k) for k in ic])
    inputs, proofs = [], []
    for _ in range(n):
        xs = [rng.randrange(R) for _ in range(n_public)]
        a, b = rng.randrange(1, R), rng.randrange(1, R)
        prep = (ic[0] + sum(x * k for x, k in zip(xs, ic[1:]))) % R
        c = (a * b - al * be - prep * ga) * pow(de, -1, R) % R
        inputs.append(xs)
        proofs.append(_proof_bytes(g1(a), g2(b), g1(c)))
    return vk, inputs, proofs


def cpp_host_rate(golden_a: int, k: int = 32):
    """proofs/s of the C++ host verify_with_processed_vk on one core, from groth16_bench (B2G_VERIFY_MANY=k, bench key)"""
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(GOLDEN, 'complex-circuit-10000-10000.zkey'), 'chain:%d' % golden_a, '0'],
                                  text=True, env=dict(os.environ, B2G_VERIFY_MANY=str(k)))
    line = [l for l in out.splitlines() if l.startswith('verify_many')][0]
    assert 'agree=1' in line, line
    return float(line.rsplit('(', 1)[1].split()[0])


def gpu_label():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True)
        return out.strip().splitlines()[0]
    except Exception as e:                                        # the numbers still stand; say where the label failed
        return f'unknown GPU ({e})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,64,1024,16384,65536')
    ap.add_argument('--keys', default='test,complex,synth100')
    ap.add_argument('--distinct', type=int, default=256)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--host-proofs', type=int, default=5)
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(',')]
    ctx = Context(0)
    print(f'# GPU: {gpu_label()}')
    makers = {'test': key_test, 'complex': key_complex, 'synth100': lambda c, n: key_synth100(c, min(n, 64))}
    for name in args.keys.split(','):
        key, inputs, proofs = makers[name](ctx, args.distinct)
        m = len(proofs)
        pvk = Groth16.process_vk(key)
        t0 = time.perf_counter()
        for k in range(args.host_proofs):
            assert Groth16.verify_with_processed_vk(pvk, inputs[k % m], proofs[k % m])
        host = args.host_proofs / (time.perf_counter() - t0)
        row = {'key': name, 'n_public': len(inputs[0]), 'distinct_proofs': m, 'host_python_proofs_per_s': round(host, 2)}
        if name == 'complex':
            a0 = int(json.load(open(os.path.join(GOLDEN, 'golden_vectors.json')))['complex_zkey']['a'])
            row['host_cpp_proofs_per_s'] = round(cpp_host_rate(a0), 2)
        for count in counts:
            xs = [inputs[k % m] for k in range(count)]
            ps = [proofs[k % m] for k in range(count)]
            assert all(Groth16.verify_many(key, xs, ps, ctx))         # warm-up (buffers, key load) and check
            best = None
            for _ in range(args.reps):
                t0 = time.perf_counter()
                Groth16.verify_many(key, xs, ps, ctx)
                dt = time.perf_counter() - t0
                best = dt if best is None else min(best, dt)
            row[f'gpu_proofs_per_s@{count}'] = round(count / best, 1)
        print(json.dumps(row), flush=True)
        release(key)
    ctx.close()


if __name__ == '__main__':
    main()
