"""Proofs/s of b2g_prove_many (one device pass for K witnesses) against the best single-proof route: three contexts kept in
flight by one host thread with b2g_prove_submit / b2g_prove_wait, witnesses in host memory.

For the squaring chain at 2^12 .. 2^20 and the reference's bench key (complex-circuit-10000-10000.zkey, 2^14), each arm is
warmed up at every count it uses, then the arms run alternately (--rounds times each) with a host clock around synchronous
calls.  Every point checks a sample of batched proofs against the single-proof bytes.  One JSON line per point goes to
stdout and, with --out, to that file; the first line records the card and its power limit.

    python tools/bench_many.py [--sizes 12,14,16,18,20] [--counts 4,16,64,256] [--rounds 2] [--out FILE]
"""
from __future__ import annotations

import argparse
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


def workloads(sizes):
    from circom_compat_b200 import synth, read_zkey, fr_to_mont
    from oracle import pyref as o
    for log_n in sizes:
        circ = synth.chain_circuit(1 << log_n)
        ws = [fr_to_mont(synth.chain_witness(1 << log_n, 3 + k)) for k in range(4)]
        yield f'chain_2^{log_n}', circ, None, circ.matrices(), ws, log_n
    pk, cm = read_zkey(open(os.path.join(ROOT, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'), 'rb').read())
    ws = [fr_to_mont(o.chain_witness(pk.n_vars, 3 + k)) for k in range(4)]
    yield 'complex-circuit-10000-10000', None, pk, cm, ws, 14


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='12,14,16,18,20')
    ap.add_argument('--counts', default='4,16,64,256')
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from circom_compat_b200 import Context, Groth16, B2gError, synth, release
    from circom_compat_b200 import _native as N
    out = open(args.out, 'w') if args.out else None

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + '\n'); out.flush()

    info = card()
    emit({'kind': 'card', **info})
    counts = [int(x) for x in args.counts.split(',')]
    inflight = [Context(0) for _ in range(3)]
    for name, circ, pk, cm, ws, log_n in workloads([int(x) for x in args.sizes.split(',')]):
        # a fresh batch context per workload: its buffers from the previous size's largest batch are not carried over.  Both
        # arms hold their device buffers at once (they alternate), so a count that does not fit beside three in-flight
        # contexts is reported with fits = false.
        ctx = Context(0)
        if pk is None:
            pk, _ = synth.setup(ctx, circ)
        r, s = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
        # proofs per timed window: enough work that one window lasts well over 100 ms at every size
        window = 256 if log_n <= 16 else 32
        single = [Groth16.create_proof_with_reduction_and_matrices(pk, r + k, s, cm, cm.num_instance_variables, cm.num_constraints, ws[k], ctx).data
                  for k in range(len(ws))]

        def inflight_arm():
            pend = {}
            t0 = time.perf_counter()
            for i in range(window):
                j = i % 3
                if j in pend:
                    pend.pop(j).wait()
                pend[j] = Groth16.submit(pk, r + i % 4, s, cm, ws[i % 4], inflight[j])
            for j in sorted(pend):
                pend[j].wait()
            return window / (time.perf_counter() - t0)

        def batch_arm(k):
            reps = max(1, window // k)
            rs = [(r + i % 4, s) for i in range(k)]
            wk = [ws[i % 4] for i in range(k)]
            t0 = time.perf_counter()
            for _ in range(reps):
                got = Groth16.create_proofs(pk, rs, cm, wk, ctx)
            rate = reps * k / (time.perf_counter() - t0)
            for i in sorted({0, k // 2, k - 1}):
                assert got[i].data == single[i % 4], (name, k, i)
            return rate

        inflight_arm()                                                    # warm-up of the three contexts first
        fits = []
        for k in counts:                                                  # warm-up: buffers, graph capture per count
            try:
                batch_arm(k); fits.append(k)
            except B2gError as e:
                if e.code != N.B2G_E_DEVICE:
                    raise
                emit({'kind': 'point', 'workload': name, 'log_n': log_n, 'arm': 'prove_many', 'count': k, 'fits': False, 'error': str(e)[:200], **info})
        rates = {'inflight3': []}
        for k in fits:
            rates[k] = []
        for _ in range(args.rounds):
            rates['inflight3'].append(inflight_arm())
            for k in fits:
                rates[k].append(batch_arm(k))
        emit({'kind': 'point', 'workload': name, 'log_n': log_n, 'arm': 'submit_wait_3_contexts', 'count': 3,
              'proofs_per_s': [round(x, 2) for x in rates['inflight3']], 'proofs_per_window': window, **info})
        for k in fits:
            emit({'kind': 'point', 'workload': name, 'log_n': log_n, 'arm': 'prove_many', 'count': k, 'fits': True,
                  'proofs_per_s': [round(x, 2) for x in rates[k]], 'proofs_per_window': max(1, window // k) * k, **info})
        release(pk); release(cm)
        ctx.close()
    for cx in inflight:
        cx.close()


if __name__ == '__main__':
    main()
