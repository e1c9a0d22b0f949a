"""Proofs/s of b2g_prove_keys (batches under K keys in one device pass) against the two routes a caller has without it:
a loop of create_proofs (b2g_prove_many) over the keys on one context, and three contexts kept in flight by one host thread
with b2g_prove_submit / b2g_prove_wait.

Each of the K keys is its own device key (a copy of one circuit's key, loaded separately), so the loop re-captures its
proof graph whenever the key changes, as it would for K circuits.  Workloads: the squaring chain at 2^12 and 2^16, the
reference's bench key (complex-circuit-10000-10000.zkey, 2^14), and a mixed group of one key each at 2^12, 2^14 and 2^16.
Every arm is warmed up at its shape, then the three arms run alternately, --rounds times each, with a host clock around
synchronous calls; the best round is the figure.  Every cell checks a sample of keyed proofs against create_proofs.  One
JSON line per cell goes to stdout and, with --out, to that file; the first line records the card and its power limit.

    python tools/bench_prove_keys.py [--workloads chain12,bench14,chain16,mixed] [--keys 1,4,16,64] [--per-key 1,4,16,64]
                                     [--rounds 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in q.split(',')]
    return {'gpu': name, 'power_limit': power, 'max_sm_clock': clock}


def circuits(ctx):
    """name -> (pk, matrices, [Montgomery witnesses])"""
    from circom_compat_b200 import synth, read_zkey, fr_to_mont
    from oracle import pyref as o
    out = {}
    for log_n in (12, 16):
        circ = synth.chain_circuit(1 << log_n)
        pk, _ = synth.setup(ctx, circ)
        out[f'chain{log_n}'] = (pk, circ.matrices(), [fr_to_mont(synth.chain_witness(1 << log_n, 3 + k)) for k in range(4)])
    pk, cm = read_zkey(open(os.path.join(ROOT, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'), 'rb').read())
    out['bench14'] = (pk, cm, [fr_to_mont(o.chain_witness(pk.n_vars, 3 + k)) for k in range(4)])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='chain12,bench14,chain16,mixed')
    ap.add_argument('--keys', default='1,4,16,64')
    ap.add_argument('--per-key', default='1,4,16,64')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from circom_compat_b200 import Context, Groth16, B2gError, release
    from circom_compat_b200 import _native as N
    out = open(args.out, 'w') if args.out else None

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + '\n'); out.flush()

    info = card()
    emit({'kind': 'card', **info})
    ctx = Context(0)
    inflight = [Context(0) for _ in range(3)]
    base = circuits(ctx)
    r, s = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    for wl in args.workloads.split(','):
        shapes = [(1, int(p)) for p in args.per_key.split(',')] if wl == 'mixed' else \
                 [(int(k), int(p)) for k in args.keys.split(',') for p in args.per_key.split(',')]
        for nk, per in shapes:
            names = ['chain12', 'bench14', 'chain16'] if wl == 'mixed' else [wl] * nk
            # every key its own device key: a shallow copy is a new host object, loaded on its own
            keys = [(copy.copy(base[n][0]), base[n][1], base[n][2]) for n in names]
            cell = {'kind': 'cell', 'workload': wl, 'keys': len(keys), 'per_key': per, **info}
            try:
                group = Groth16.load_proving_keys([(pk, cm) for pk, cm, _ in keys], ctx)
            except B2gError as e:
                emit({**cell, 'refused': str(e)[:200]}); continue
            batches = [([(r + i, s) for i in range(per)], [ws[i % 4] for i in range(per)]) for _, _, ws in keys]

            def keyed():
                return Groth16.create_proofs_keys(group, batches, ctx)

            def loop():
                return [Groth16.create_proofs(pk, rs, cm, ws, ctx) for (pk, cm, _), (rs, ws) in zip(keys, batches)]

            def contexts():
                pend, got, i = {}, [], 0
                for (pk, cm, _), (rs, ws) in zip(keys, batches):
                    for (ri, si), w in zip(rs, ws):
                        j = i % 3
                        if j in pend:
                            got.append(pend.pop(j).wait())
                        pend[j] = Groth16.submit(pk, ri, si, cm, w, inflight[j])
                        i += 1
                for j in sorted(pend):
                    got.append(pend[j].wait())
                return got

            total = len(keys) * per
            rates = {'prove_keys': [], 'loop_create_proofs': [], 'inflight3': []}
            try:
                got = keyed()
                ref = loop()
                contexts()
                assert [[p.data for p in b] for b in got] == [[p.data for p in b] for b in ref], (wl, nk, per)
                for _ in range(args.rounds):
                    for arm, fn in (('prove_keys', keyed), ('loop_create_proofs', loop), ('inflight3', contexts)):
                        t0 = time.perf_counter()
                        fn()
                        rates[arm].append(total / (time.perf_counter() - t0))
            except B2gError as e:
                if e.code not in (N.B2G_E_DEVICE, N.B2G_E_SHAPE):
                    raise
                emit({**cell, 'refused': str(e)[:200]})
            else:
                emit({**cell, 'proofs': total, **{arm: round(max(v), 1) for arm, v in rates.items()},
                      'rounds': {arm: [round(x, 1) for x in v] for arm, v in rates.items()}})
            release(group)
            for pk, _, _ in keys:
                release(pk)
    for cx in inflight + [ctx]:
        cx.close()


if __name__ == '__main__':
    main()
