"""Preparing a ceremony for phase 2 (b2g_powers_prepare) and what a prepared file saves.

1. Groth16.prepare_powers_of_tau on an honest ceremony at each --prepare power (made by fixed-base products), best of --reps
   (the first call includes module loading, so --reps 1 overstates the small powers).
2. The setup from the prepared ceremony (b2g_setup_from_lagrange) against the transform route (b2g_setup_from_powers) at
   each --setup size, for the chain and circomlike circuits under both reductions, alternating; the two keys are compared
   byte for byte in the same run.
3. verify_powers_of_tau on the prepared ceremony against the same ceremony without its Lagrange sections, alternating.
The card name and power limit are read in the same command.

    python tools/bench_ptau_prepare.py [--prepare 12,16,18,20,22] [--setup 14,16,18,20] [--verify 20] [--reps 3]
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

from bench_ptau_check import alternate, ceremony  # noqa: E402
from bench_verify import gpu_label  # noqa: E402
from circom_compat_b200 import CircomReduction, Context, Groth16, LibsnarkReduction, Powers, synth  # noqa: E402
from circom_compat_b200.zkey import R_MOD  # noqa: E402

KEY_FIELDS = ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'delta_g1', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query',
              'b_g2_query', 'l_query', 'h_query')


def same_key(a, b) -> bool:
    return all(np.ascontiguousarray(getattr(a, k)).tobytes() == np.ascontiguousarray(getattr(b, k)).tobytes() for k in KEY_FIELDS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--prepare', default='12,16,18,20,22')
    ap.add_argument('--setup', default='14,16,18,20')
    ap.add_argument('--verify', default='20')
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    sizes = lambda s: [int(x) for x in s.split(',') if x]
    prep_p, setup_p, verify_p = sizes(args.prepare), sizes(args.setup), sizes(args.verify)
    ctx = Context(0)
    print(json.dumps({'gpu': gpu_label()}), flush=True)
    top = max(prep_p + setup_p + verify_p)
    rng = random.Random(0xB2)
    big = ceremony(ctx, top, *(rng.randrange(1, R_MOD) for _ in range(3)))
    prepared = {}
    for p in sorted(set(prep_p + setup_p + verify_p)):
        pre = big.prefix(p, copy=True)
        best = None
        for _ in range(args.reps if p in prep_p else 1):
            t0 = time.perf_counter()
            out = Groth16.prepare_powers_of_tau(pre, ctx=ctx, power=p)
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        prepared[p] = (pre, out)
        if p in prep_p:
            print(json.dumps({'bench': 'prepare', 'power': p, 's': round(best, 4)}), flush=True)
    for p in setup_p:
        pre, out = prepared[p]
        for kind in ('chain', 'circomlike'):
            circ = synth.chain_circuit(1 << p) if kind == 'chain' else synth.circomlike_circuit(p)[0]
            for red in (CircomReduction, LibsnarkReduction):
                res = alternate(args.reps, {
                    'lagrange': lambda: Groth16.generate_parameters_from_powers_of_tau(circ, out, ctx, red),
                    'transform': lambda: Groth16.generate_parameters_from_powers_of_tau(circ, pre, ctx, red)})
                print(json.dumps({'bench': 'setup', 'log_n': p, 'circuit': kind, 'reduction': red.__name__,
                                  'lagrange_s': round(res['lagrange'][1], 4), 'transform_s': round(res['transform'][1], 4),
                                  'identical': same_key(res['lagrange'][0], res['transform'][0])}), flush=True)
    for p in verify_p:
        pre, out = prepared[p]
        plain = Powers(out.power, out.ceremony_power, out.tau_g1, out.tau_g2, out.alpha_tau_g1, out.beta_tau_g1, out.beta_g2)
        res = alternate(args.reps, {'prepared': lambda: bool(Groth16.verify_powers_of_tau(out, ctx=ctx)),
                                    'unprepared': lambda: bool(Groth16.verify_powers_of_tau(plain, ctx=ctx))})
        print(json.dumps({'bench': 'verify', 'power': p, 'prepared_s': round(res['prepared'][1], 4),
                          'unprepared_s': round(res['unprepared'][1], 4),
                          'verdicts': [res['prepared'][0], res['unprepared'][0]]}), flush=True)
    ctx.close()


if __name__ == '__main__':
    main()
